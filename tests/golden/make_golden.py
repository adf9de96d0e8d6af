"""Generates the committed golden fixtures from the UNMODIFIED reference
(/root/reference/src/sniffles behind oracle/pyref's stub pysam).  Runs only in the build
container; the fixtures travel, the reference does not.

    python tests/golden/make_golden.py

Writes tests/golden/<name>.json (reference outputs for a seeded synthetic block: the lead
table before clustering, the candidates as they leave Task.call_candidates, the finalized
calls with FILTER / GT / ALT) and tests/golden/hg008_bnd.npz + .json (the reference's own
test BAMs src/tests/data/hg008.bam, hg002.bam packed into a record block, with what
Lead.for_bnd returns per record — the vectors of src/tests/test_bnd_leads.py)."""
import hashlib
import json
import logging
import os
import platform
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref")]
logging.disable(logging.CRITICAL)

import harness  # noqa: E402
from sniffles_b200 import bamio, synth  # noqa: E402

FIXTURES = {
    # name: (synth.generate kwargs, reference CLI args)
    "c1_ont_1mb": (dict(seed=1001, contig_len=[1_000_000], coverage=20.0, len_model=0, len_mean=100000.0, len_sd=10000.0,
                        len_min=1000, len_max=200000, tech="ont", sv_spacing=25000.0), []),
    "c2_ont_wgs_small": (dict(seed=1002, contig_len=[300_000, 260_000, 220_000, 150_000], coverage=30.0, len_model=1, len_mean=15000.0,
                              len_sd=600.0, tech="ont", sv_spacing=15000.0), []),
    "c3_hifi_mosaic": (dict(seed=1003, contig_len=[400_000, 300_000], coverage=60.0, len_model=0, len_mean=18000.0, len_sd=3000.0,
                            len_max=60000, tech="hifi", mosaic=True, sv_spacing=12000.0), ["--mosaic"]),
    "c5_ins_heavy": (dict(seed=1005, contig_len=[150_000], coverage=20.0, len_model=0, len_mean=20000.0, len_sd=2000.0, len_min=5000,
                          len_max=60000, tech="ont", sv_spacing=1000.0, ins_only=True, tr_frac=0.0, clip_prob=0.0), []),
    "tr_repeat_noqc": (dict(seed=77, contig_len=[250_000], coverage=25.0, len_mean=9000.0, len_sd=2500.0, tech="ont", sv_spacing=2500.0,
                            tr_frac=0.6, clip_prob=0.3, phased_frac=1.0), ["--no-qc"]),
    "auto_support_qcnm": (dict(seed=78, contig_len=[200_000, 180_000], coverage=40.0, len_mean=6000.0, len_sd=1500.0, tech="ont",
                               sv_spacing=4000.0, lowmapq_prob=0.3, phased_frac=0.0), ["--minsupport", "auto", "--qc-nm"]),
    "phased_phase": (dict(seed=79, contig_len=[260_000, 140_000], coverage=30.0, len_mean=12000.0, len_sd=3000.0, tech="ont", sv_spacing=5000.0,
                          phased_frac=0.8, tr_frac=0.1, clip_prob=0.2), ["--phase"]),
    # the next three pin the oracle only (the GPU golden test lists its fixtures explicitly)
    "filters_binsize": (dict(seed=80, contig_len=[220_000], coverage=35.0, len_mean=8000.0, len_sd=2500.0, tech="ont", sv_spacing=3000.0,
                             lowmapq_prob=0.25, clip_prob=0.3), ["--mapq", "30", "--min-alignment-length", "3000", "--cluster-binsize", "50", "--cluster-r", "1.5"]),
    "long_ins_minsv": (dict(seed=81, contig_len=[240_000], coverage=25.0, len_mean=25000.0, len_sd=5000.0, len_max=80000, tech="ont", sv_spacing=6000.0,
                            sv_min=30, sv_max=9000, clip_prob=0.4), ["--minsvlen", "30", "--long-ins-length", "1500", "--minsupport", "3"]),
    "hifi_strict": (dict(seed=82, contig_len=[200_000, 120_000], coverage=45.0, len_mean=16000.0, len_sd=2000.0, len_max=40000, tech="hifi", sv_spacing=4000.0,
                         phased_frac=0.5, tr_frac=0.3), ["--cluster-merge-pos", "80", "--cluster-merge-len", "0.2", "--no-consensus"]),
}


MASKS = {"c2_ont_wgs_small": {0: [(20_000, 26_000), (150_000, 150_700)], 2: [(0, 5_000), (219_000, 220_000)]}}   # reference 'N' runs (A8)


def block_digest(blk):
    h = hashlib.sha256()
    for a in (blk.rec, blk.cigar, blk.var, blk.seq, blk.task, blk.tr):
        h.update(np.ascontiguousarray(a).tobytes())
    return h.hexdigest()


def make_synthetic(only=None):
    for name, (kw, args) in FIXTURES.items():
        if only and name not in only:
            continue
        kw2 = dict(kw)
        blk = synth.generate(kw2.pop("seed"), kw2.pop("contig_len"), kw2.pop("coverage"), **kw2)
        if name in MASKS:
            blk.set_n_mask(MASKS[name])
        cfg = harness.make_config(*args)
        tasks = [harness.run_task(blk, t, cfg) for t in range(len(blk.task))]
        out = dict(generator=kw, args=args, n_mask={str(k): v for k, v in MASKS.get(name, {}).items()}, digest=block_digest(blk), n_rec=len(blk.rec), tasks=tasks,
                   made_with=dict(python=platform.python_version(), numpy=np.__version__, reference="fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867"))
        path = os.path.join(HERE, name + ".json")
        with open(path, "w") as f:
            json.dump(out, f, separators=(",", ":"))
        print(name, "records", len(blk.rec), "cands", sum(len(t["cands"]) for t in tasks), os.path.getsize(path) // 1024, "KiB")


def make_bam_vectors():
    harness.import_reference()
    from sniffles.leadprov import Lead
    data = os.path.join(harness.REFERENCE_SRC, "tests", "data")
    blocks, expect = [], []
    for fn in ("hg008.bam", "hg002.bam"):
        f = bamio.BamFile(os.path.join(data, fn))
        tasks, recs = [], []                # one task per contig that has records ([0, len-1], as the reference plans them: sniffles:313-358)
        for c, (name, length) in enumerate(f.contigs):
            got = list(f.fetch(name, 0, length))
            if got:
                recs.extend((len(tasks), r) for r in got)
                tasks.append((c, 0, length - 1, len(tasks)))
        blk = bamio.pack_records(f.contigs, recs, tasks, with_seq=False)
        f.close()
        for i in range(len(blk.rec)):
            rd = harness.DuckRead(blk, i)
            ld = Lead.for_bnd(0, rd)
            expect.append(dict(file=fn, qname=rd.query_name, contig=rd.reference_name, pos=rd.reference_start,
                               lead=None if ld is None else [ld.ref_start, ld.bnd_info.mate_contig, ld.bnd_info.mate_ref_start,
                                                             bool(ld.bnd_info.is_first), bool(ld.bnd_info.is_reverse)]))
        blocks.append((fn, blk))
    arrays = {}
    for fn, blk in blocks:
        k = fn.split(".")[0]
        for nm in ("rec", "cigar", "var", "task", "contig"):
            arrays[f"{k}_{nm}"] = getattr(blk, nm)
        arrays[f"{k}_names"] = np.array(blk.contig_names)
    np.savez_compressed(os.path.join(HERE, "hg008_bnd.npz"), **arrays)
    with open(os.path.join(HERE, "hg008_bnd.json"), "w") as f:
        json.dump(dict(source="src/tests/data/hg008.bam, hg002.bam; expectations = Lead.for_bnd of the reference at HEAD "
                              "(8 leads equal the tuples asserted in src/tests/test_bnd_leads.py:48-188, 9 are None)", records=expect), f, indent=1)
    print("bam vectors", [(e["qname"][:8], e["lead"]) for e in expect])


def make_config_dump():
    out = {}
    for args in ([], ["--mosaic"], ["--no-qc"], ["--minsvlen", "30"], ["--minsupport", "auto"], ["--dev-no-qc"], ["--qc-nm", "--cluster-merge-len", "0.3"]):
        cfg = harness.make_config(*args)
        out[" ".join(args)] = {k: v for k, v in vars(cfg).items() if isinstance(v, (int, float, str, bool, type(None))) and k not in
                               ("start_date", "run_id", "command", "workdir", "tmp_dir", "version", "build", "snf_format_version", "input", "vcf")}
    with open(os.path.join(HERE, "config_defaults.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)


def make_snf():
    """the reference's own .snf for one fixture block (the SNF reader / writer are pinned against it)"""
    kw, args = FIXTURES["c2_ont_wgs_small"]
    kw2 = dict(kw)
    blk = synth.generate(kw2.pop("seed"), kw2.pop("contig_len"), kw2.pop("coverage"), **kw2)
    path = os.path.join(HERE, "c2_ont_wgs_small.snf")
    harness.write_reference_snf(blk, args, path)
    print("snf", os.path.getsize(path) // 1024, "KiB")


def make_local_asm_vectors():
    """the reference's own LocalAsm.select_padding / solve_ins / solve_del / SPOA.set on seeded alignment strings
    (local_asm.py:26-252): pins the host side of the local assembly; the POA itself (pyspoa) is absent here"""
    import random
    import types
    harness.import_reference()
    from sniffles import local_asm
    rnd = random.Random(2024)
    out = dict(padding=[], scores=[], solve=[])
    for svlen in [45, 50, 120, 399, 400, 401, 800, 1200, 1201, 3000, 9999, 10000, -60, -400, -401, -5000]:
        sv = types.SimpleNamespace(svlen=svlen)
        la = local_asm.LocalAsm.__new__(local_asm.LocalAsm)
        la.sv = sv
        out["padding"].append([svlen, la.select_padding("sv"), la.select_padding("half")])
        sp = local_asm.SPOA()
        sp.set(svlen)
        out["scores"].append([svlen, sp.match, sp.miss, sp.gap_open, sp.gap_expand, sp.gap_open2, sp.gap_expand2])
    bases = "ACGT"
    for k in range(240):
        svtype = "INS" if k % 2 == 0 else "DEL"
        svlen = rnd.choice([50, 80, 150, 400, 900, 2000])
        L = rnd.randrange(200, 1500)
        core = "".join(rnd.choice(bases) for _ in range(L))
        cut = rnd.randrange(20, L - 20)
        gap = max(1, int(svlen * rnd.choice([0.5, 0.86, 0.95, 1.0, 1.05, 1.14, 1.3])))
        extra = rnd.choice([0, 0, 1, 2, 4])            # more small gap runs somewhere
        insseq = "".join(rnd.choice(bases) for _ in range(gap))
        if svtype == "INS":
            sv_aln, ref_aln = core[:cut] + insseq + core[cut:], core[:cut] + "-" * gap + core[cut:]
        else:
            sv_aln, ref_aln = core[:cut] + "-" * gap + core[cut:], core[:cut] + insseq + core[cut:]
        for _ in range(extra):
            p = rnd.randrange(5, len(sv_aln) - 5)
            g = rnd.randrange(1, 6)
            if rnd.random() < 0.5:
                sv_aln, ref_aln = sv_aln[:p] + "-" * g + sv_aln[p:], ref_aln[:p] + "".join(rnd.choice(bases) for _ in range(g)) + ref_aln[p:]
            else:
                sv_aln, ref_aln = sv_aln[:p] + "".join(rnd.choice(bases) for _ in range(g)) + sv_aln[p:], ref_aln[:p] + "-" * g + ref_aln[p:]
        ref_pos = rnd.choice([0, 1000, 123456])
        sv = types.SimpleNamespace(svlen=svlen if svtype == "INS" else -svlen, svtype=svtype)
        la = local_asm.LocalAsm.__new__(local_asm.LocalAsm)
        la.sv = sv
        region = f"ctg1:{ref_pos}-{ref_pos + 5000}"
        res = la.solve_ins(region, sv_aln, ref_aln) if svtype == "INS" else la.solve_del(region, sv_aln, ref_aln)
        out["solve"].append(dict(svtype=svtype, svlen=sv.svlen, ref_pos=ref_pos, sv_aln=sv_aln, ref_aln=ref_aln, want=[res[0], res[1], bool(res[2])]))
    with open(os.path.join(HERE, "local_asm", "vectors.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))
    print("local_asm vectors", len(out["solve"]), "accepted", sum(v["want"][2] for v in out["solve"]))


if __name__ == "__main__":
    if sys.argv[1:] == ["lasm"]:
        make_local_asm_vectors()
        sys.exit(0)
    if sys.argv[1:] == ["snf"]:
        make_snf()
        sys.exit(0)
    if len(sys.argv) > 1:
        make_synthetic(set(sys.argv[1:]))
        sys.exit(0)
    make_config_dump()
    make_synthetic()
    make_bam_vectors()
