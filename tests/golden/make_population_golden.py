"""Generates the population golden data: population SNFs under tests/golden/population/ and, for combine runs with
--combine-population, the whole VCF the UNMODIFIED reference writes (expected.json) plus the index its get_population_AF picks for a
seeded set of queries (match_vectors.json).

  * P4, P4_all, P_ctg1: written by the reference's own PopulationSNF through CombineResultTmpFilePopulationSNF and write_results, with the
    setup of sniffles:272-279, 463-464 and 566-568 restated (the `sniffles` entry forks workers, which the build container's stubs do not
    serve): s1..s4 of tests/combine_cli_common.py with defaults, with --dev-population-min-gt 0, and with --contig ctg1.
  * P_edit: P4_all's variants with deterministic edits, rewritten with the reference's classes (SNFileBase.store, write_and_index,
    write_results): INS ALTs replaced so that they fail only the alignment test, duplicated variants (equal-distance ties), variants moved
    across a block edge, INS ALTs longer than 2,048 bytes, and one block listed in two parts (only the first is read).
  * expected.json: the combine cases below, run as make_combine_cli_golden runs them, except that every task gets a pickled copy of the
    config, as the reference's pipe delivers it (CombineTask.execute replaces config.combine_population by the opened file).  Each case
    counts its calls by class, from an instrumented get_population_AF.
  * match_vectors.json: per parameter set, the file-order index get_population_AF picks for the queries population_common.seeded_queries
    draws from P_edit: every variant's af is set to its index in the loaded blocks, so the value the reference's loop returns names the
    variant; -2 where it raises ZeroDivisionError.
Run in the build container (needs /root/reference):
    python tests/golden/make_population_golden.py"""
import io
import json
import os
import pickle
import random
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle", "pyref"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import combine_cli_common as ccc                   # noqa: E402
import population_common as pc                     # noqa: E402
import harness                                     # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "population")
S4 = ["s1.snf", "s2.snf", "s3.snf", "s4.snf"]
TYPES = ["INS", "DEL", "DUP", "INV", "BND"]
CONTIGS = ["ctg1", "ctg2"]

# (label, inputs, extra arguments, population SNF)
CASES = [
    ("two", ["s1.snf", "s2.snf"], [], "P4"),
    ("default4", S4, [], "P4_all"),
    ("no_alignment4", S4, ["--combine-pctseq", "0"], "P_edit"),
    ("strict_alignment4", S4, ["--combine-pctseq", "0.985", "--combine-separate-intra"], "P_edit"),
    ("loose4", S4, ["--combine-match", "100", "--combine-low-confidence", "0.6", "--combine-output-filtered"], "P_edit"),
    ("contig_absent", S4, ["--contig", "ctg2"], "P_ctg1"),
    ("regions", ["s1.snf", "s2.snf", "s3.snf"], ["--regions", "regions.bed"], "P_edit"),
    ("tmpfile", S4, ["--combine-max-inmemory-results", "1"], "P_edit"),
    ("phase", S4, ["--phase"], "P4"),
]
CLASSES = ("ins_aligned_match", "ins_alignment_rejected", "ins_match_no_alignment", "non_ins_match", "unmatched", "contig_absent")


def _setup(paths, extra, tmp):
    """the combine-mode setup of sniffles:371-481 (as make_combine_cli_golden restates it) -> (config, contig_lengths, tasks, result_class)"""
    harness.import_reference()
    from sniffles import parallel, snf as refsnf
    from sniffles.config import SnifflesConfig
    config = SnifflesConfig("--input", *paths, "--vcf", os.path.join(tmp, "out.vcf"), "--tmp-dir", tmp, *extra)
    config.mode = "combine"
    config.snf_input_info, config.sample_ids_vcf = [], []
    for internal_id, fn in enumerate(paths):
        snf_in = refsnf.SNFile(config, open(fn, "rb"), filename=fn)
        snf_in.read_header()
        contig_lengths = snf_in.header["config"]["contig_lengths"]
        sample_id = snf_in.header["config"]["sample_id"] if snf_in.header["config"]["sample_id"] is not None else os.path.splitext(os.path.basename(fn))[0]
        config.snf_input_info.append({"internal_id": internal_id, "sample_id": sample_id, "filename": fn})
        snf_in.close()
    for info in config.snf_input_info:
        config.sample_ids_vcf.append((info["internal_id"], info["sample_id"]))
    if to_process := (config.contig or config.regions_by_contig):
        contig_lengths = [(name, length) for name, length in contig_lengths if name in to_process]
    result_class = None
    if len(paths) > config.combine_max_inmemory_results:
        from sniffles.result import CombineResultTmpFile
        result_class = CombineResultTmpFile
    if config.dev_population_snf:                    # sniffles:463-464
        from sniffles.result import CombineResultTmpFilePopulationSNF
        result_class = CombineResultTmpFilePopulationSNF
    tasks, task_id = [], 0
    for contig_str, contig_length in contig_lengths:
        task = parallel.CombineTask(id=task_id, contig=contig_str, start=0, end=contig_length - 1, assigned_process_id=None, sv_id=0,
                                    config=config, result_class=result_class, regions=config.regions_by_contig.get(contig_str))
        tasks.extend(task.scatter())
        task_id = tasks[-1].id + 1
    for t in tasks:                                  # each task reaches its worker pickled, with a config of its own
        t.config = pickle.loads(pickle.dumps(config))
    return config, contig_lengths, tasks, result_class


def write_population_snf(paths, extra, out_path, tmp):
    """sniffles:272-279, 463-464, 566-568: the reference's population SNF of a combine run"""
    from sniffles import vcf as refvcf
    from sniffles.snfp import PopulationSNF
    config, contig_lengths, tasks, _ = _setup(paths, ["--dev-population-snf", out_path, *extra], tmp)
    psnf_out = PopulationSNF(config, open(out_path, "wb"))
    vcf_out = refvcf.VCF(config, io.StringIO())
    for t in tasks:
        t.result = t.execute()
        t.result.emit(vcf_out=vcf_out, psnf_out=psnf_out)
    n = psnf_out.write_results(config, [name for name, _ in contig_lengths])
    psnf_out.close()
    return n


def edited_population(src, out_path, tmp):
    """P_edit: the variants of `src` with deterministic edits, written by the reference's classes"""
    from sniffles.config import SnifflesConfig
    from sniffles.snf import SNFileBase
    from sniffles.snfp import PopulationSNF
    config = SnifflesConfig("--input", "x.snf", "--vcf", os.path.join(tmp, "x.vcf"), "--tmp-dir", tmp, "--dev-population-snf", out_path)
    config.snf_input_info = [{"internal_id": k, "sample_id": f"s{k}", "filename": f"s{k}.snf"} for k in range(4)]
    psnf = PopulationSNF.open(src)
    rng = random.Random(20261017)
    bs = config.snf_block_size
    per_contig = {}
    for contig in CONTIGS:
        out = []
        for block, blk in psnf.get_all_blocks(contig).items():
            for t in TYPES:
                out.extend(blk[t])
        per_contig[contig] = out
    psnf.close()
    edits = {"alignment_only": 0, "tie": 0, "block_edge": 0, "long_alt": 0, "zero_len_ins": 0}
    for contig, vs in per_contig.items():
        new = []
        for i, v in enumerate(vs):
            if v.svtype == "INS" and v.alt and not v.alt.startswith("<") and i % 5 == 1:
                v.alt = "".join(rng.choice("ACGT") for _ in v.alt)            # same length: passes the position test, fails the alignment
                edits["alignment_only"] += 1
            elif v.svtype == "INS" and i % 11 == 4:
                v.alt = "".join(rng.choice("ACGT") for _ in range(2048 + rng.randrange(1500)))
                v.svlen = len(v.alt)
                edits["long_alt"] += 1
            elif i % 7 == 3:                                                  # a block edge within 40 bp, on either side
                edge = (v.pos // bs + (1 if v.pos % bs >= bs // 2 else 0)) * bs
                if edge > 0:
                    v.pos = edge + rng.randrange(-40, 40)
                    v.end = v.pos + (abs(v.svlen) if v.svtype != "INS" else 0)
                    edits["block_edge"] += 1
            new.append(v)
            if i % 6 == 2:                                                    # an equal-distance twin right after it
                twin = pickle.loads(pickle.dumps(v))
                twin.id, twin.af, twin.genotyped_sample_count = v.id + "_twin", round(1.0 - v.af, 6), v.genotyped_sample_count + 1
                new.append(twin)
                edits["tie"] += 1
        per_contig[contig] = new
    # a zero-length INS far from every call (the division by zero of PopulationVariant.match; matched only at distance 0)
    z = pickle.loads(pickle.dumps(next(v for v in per_contig["ctg2"] if v.svtype == "INS")))
    z.id, z.pos, z.svlen, z.end, z.alt = "zero_len_ins", 259_990, 0, 259_990, ""
    per_contig["ctg2"].append(z)
    edits["zero_len_ins"] += 1
    results = []
    task_id = 0
    for contig, vs in per_contig.items():
        parts = [vs]
        if contig == "ctg1":                                                  # one block in two parts: the second is never read
            first_block = int(vs[0].pos / bs) * bs
            extra = [pickle.loads(pickle.dumps(v)) for v in vs if int(v.pos / bs) * bs == first_block]
            for v in extra:
                v.id, v.af, v.genotyped_sample_count = v.id + "_part2", 0.99999, 999
            parts.append(extra)
        for part in parts:
            fn = os.path.join(tmp, f"pedit-{task_id}.part.snf")
            p = PopulationSNF(config, open(fn, "wb"))
            for v in part:
                SNFileBase.store(p, v)
            p.write_and_index()
            p.close()
            results.append(types.SimpleNamespace(has_snf=True, task_id=task_id, contig=contig, snf_index=p.get_index(), snf_total_length=p.get_total_length(),
                                                 snf_filename=fn, snf_candidate_count=len(part), coverage_average_total=0))
            task_id += 1
    out = PopulationSNF(config, open(out_path, "wb"))
    for r in results:
        out.add_result(r)
    n = out.write_results(config, CONTIGS)
    out.close()
    return n, edits


def annotated_vcf(paths, extra, population, tmp, counts):
    """the combine VCF of the reference with --combine-population"""
    from sniffles import vcf as refvcf
    config, contig_lengths, tasks, result_class = _setup(paths, [*extra, "--combine-population", population], tmp)
    buf = io.StringIO()
    vcf_out = refvcf.VCF(config, buf)
    vcf_out.write_header(contig_lengths)
    unsorted = 0
    for t in tasks:
        t.result = t.execute()
        if result_class is not None and os.path.exists(t.result.tmpfile_unsorted):
            with open(t.result.tmpfile_unsorted) as f:
                unsorted += sum(1 for _ in f)
            os.unlink(t.result.tmpfile_unsorted)
        t.result.emit(vcf_out=vcf_out)
    return ccc.vcf_lines(buf.getvalue()), unsorted


def instrument(counts):
    """wraps PopulationSNF.get_population_AF to count the calls by class (the reference's own result is returned unchanged)"""
    from sniffles import snfp
    from sniffles.config import SnifflesConfig
    orig = snfp.PopulationSNF.get_population_AF
    if getattr(orig, "_counted", False):
        orig = orig._orig

    def counted(self, svcall):
        res = orig(self, svcall)
        cfg = SnifflesConfig.GLOBAL
        if svcall.contig not in self.index:
            cls = "contig_absent"
        elif res is not None:
            cls = ("ins_aligned_match" if cfg.combine_pctseq else "ins_match_no_alignment") if svcall.svtype == "INS" else "non_ins_match"
        else:
            cls = "unmatched"
            if svcall.svtype == "INS" and cfg.combine_pctseq:
                block = str(self._calculate_block_index(svcall.pos))
                for pv in self._blocks.get(svcall.contig, {}).get(block, {}).get("INS", []):
                    dist = abs(pv.pos - svcall.pos) + abs(abs(pv.svlen) - abs(svcall.svlen))
                    if not (dist > cfg.combine_match * float(min(abs(pv.svlen), abs(svcall.svlen))) ** 0.5 or dist > cfg.combine_match_max):
                        cls = "ins_alignment_rejected"
                        break
        counts[cls] = counts.get(cls, 0) + 1
        return res
    counted._counted, counted._orig = True, orig
    snfp.PopulationSNF.get_population_AF = counted


def match_vectors(p_edit, tmp):
    """seeded queries against P_edit; per parameter set the index the reference's get_population_AF picks"""
    from sniffles.config import SnifflesConfig
    from sniffles.snfp import PopulationSNF
    SnifflesConfig("--input", "x.snf", "--vcf", os.path.join(tmp, "x.vcf"))
    psnf = PopulationSNF.open(p_edit)
    flat = []
    for contig in CONTIGS:
        psnf._blocks[contig] = psnf.get_all_blocks(contig)
        for block, blk in psnf._blocks[contig].items():
            for t in TYPES:
                flat.extend(blk[t])
    for i, v in enumerate(flat):                     # the af the loop returns names the variant
        v.af = float(i)
    n, seed = 2000, 7
    q = pc.seeded_queries([v.contig for v in flat], [v.svtype for v in flat], [v.pos for v in flat], [v.svlen for v in flat],
                          [(v.alt or "").encode("latin-1") for v in flat], n, seed)
    queries = [dict(contig=c, svtype=t, pos=p, svlen=sl, alt=a.decode("latin-1")) for c, t, p, sl, a in zip(*q.values())]
    params = [{"combine_match": 250, "combine_match_max": 1000, "combine_pctseq": 0.7}, {"combine_match": 250, "combine_match_max": 1000, "combine_pctseq": 0.0},
              {"combine_match": 500, "combine_match_max": 150, "combine_pctseq": 0.3}]
    out = {"contigs": CONTIGS, "n": n, "seed": seed, "sets": []}
    for prm in params:
        cfg = SnifflesConfig("--input", "x.snf", "--vcf", os.path.join(tmp, "x.vcf"), "--combine-match", str(prm["combine_match"]),
                             "--combine-match-max", str(prm["combine_match_max"]), "--combine-pctseq", str(prm["combine_pctseq"]))
        psnf.config = cfg
        best = []
        for q in queries:
            try:
                res = psnf.get_population_AF(types.SimpleNamespace(**q))
            except ZeroDivisionError:
                best.append(-2)
                continue
            best.append(-1 if res is None else int(res[0]))
        out["sets"].append({**prm, "best": best})
    psnf.close()
    return out


def main():
    os.makedirs(OUT, exist_ok=True)
    gold = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via tests/golden/make_population_golden.py", "headers": [], "records": [],
            "cases": {}, "populations": {}}
    pools = {"headers": {}, "records": {}}

    def index(kind, item):
        key = json.dumps(item)
        if key not in pools[kind]:
            pools[kind][key] = len(gold[kind])
            gold[kind].append(item)
        return pools[kind][key]
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(ccc.write_inputs(os.path.join(tmp, "in")))
        harness.import_reference()
        for name, files, extra in (("P4", S4, []), ("P4_all", S4, ["--dev-population-min-gt", "0"]), ("P_ctg1", S4, ["--contig", "ctg1"])):
            d = os.path.join(tmp, "w_" + name)
            os.makedirs(d)
            n = write_population_snf(files, extra, os.path.join(OUT, name + ".snf"), d)
            gold["populations"][name] = {"inputs": files, "args": extra, "variants": n}
            print(name, "variants", n, flush=True)
        d = os.path.join(tmp, "w_P_edit")
        os.makedirs(d)
        n, edits = edited_population(os.path.join(OUT, "P4_all.snf"), os.path.join(OUT, "P_edit.snf"), d)
        gold["populations"]["P_edit"] = {"from": "P4_all", "variants": n, "edits": edits}
        print("P_edit variants", n, edits, flush=True)
        for label, files, extra, pop in CASES:
            d = os.path.join(tmp, label)
            os.makedirs(d)
            counts = {}
            instrument(counts)
            lines, unsorted = annotated_vcf(files, extra, os.path.join(OUT, pop + ".snf"), d, counts)
            gold["cases"][label] = {"inputs": files, "args": extra, "population": pop, "dropped": unsorted, "classes": {k: counts.get(k, 0) for k in CLASSES},
                                    "headers": [index("headers", x) for x in lines if isinstance(x, str)],
                                    "records": [index("records", x) for x in lines if not isinstance(x, str)]}
            print(label, "records", sum(not isinstance(x, str) for x in lines), counts, flush=True)
        vectors = match_vectors(os.path.join(OUT, "P_edit.snf"), tmp)
    with open(os.path.join(OUT, "expected.json"), "w") as f:
        json.dump(gold, f, separators=(",", ":"))
    with open(os.path.join(OUT, "match_vectors.json"), "w") as f:
        json.dump(vectors, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
