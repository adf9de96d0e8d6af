"""Generates the committed force-calling fixtures from the UNMODIFIED reference (/root/reference/src/sniffles behind oracle/pyref's stub
pysam).  Runs only in the build container; the fixtures travel, the reference does not.

    python tests/golden/make_genotype_golden.py

1. Parser / rewrite: tests/golden/genotype/<name>.vcf run through VCF.read_svs_iter, VCF.rewrite_header_genotype and
   VCF.rewrite_genotype (vcf.py:352-478) with a fixed genotype per record -> expected.json (or the fatal error's message).
2. Force calling: for four record blocks (three synthetic call fixtures and the reference's hg008 BND BAM) a target VCF derived from the
   block's own reference candidates, run through the unmodified GenotypeTask.execute (parallel.py:300-369) per planned task -- the
   lead_provider is prebuilt from DuckBam and only the instance's build_leadtab is replaced -- and written by GenotypeResult.emit in task
   order; a task that raises is left out, as the worker leaves it out -> tests/golden/genotype/<block>.targets.vcf + <block>.expected.json.
The reference's own SnifflesConfig supplies every default (genotype_format, phase, genotype_none)."""
import io
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, "genotype")
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests")]

import harness  # noqa: E402

STAMP = {"command": "sniffles --input sample.bam --genotype-vcf targets.vcf --vcf out.vcf", "start_date": "2026/10/16 00:00:00",
         "version": "Sniffles2", "build": "2.6.3"}

HEAD = ("##fileformat=VCFv4.2\n##contig=<ID=chr1,length=248956422>\n"
        '##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">\n'
        "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE\n")
REC = ["chr1\t1001\tid1\tN\t<INS>\t60\tPASS\tSVTYPE=INS;SVLEN=300;END=1001\tGT\t0/1",
       "chr1\t5000\tid2\tACGTACGTAC\tA\t.\tPASS\tPRECISE\tGT\t1/1",                 # no SVTYPE / SVLEN: DEL from REF / ALT
       "chr1\t9501\tid3\tN\t<DUP>\t12\tGT\tSVTYPE=DUP;SVLEN=0;END=9501\tGT\t0/1",
       "chr1\t10\tid4\tN\t<CNV>\t5\tPASS\tSVTYPE=CNV;SVLEN=-2000;END=2010",
       "chr1\t20000\tid5\tN\tN[chr2:5000[\t60\tPASS\tSVTYPE=TRA\tGT:DR\t0/1:3",
       "chr1\t20010\tid6\tN\t]chrUn_x:77]N\t60\tPASS\tSVTYPE=BND;CHR2=chrUn_x\tGT\t0/1",
       "chr1\t1\tid7\tA\tAGGGGGGGGGGG\t60\tPASS\tIMPRECISE;SVTYPE=INS",                # POS 1 -> pos 0; svlen len(ALT)
       "chr1\t0\tid8\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL;SVLEN=-120;END=120",            # POS 0 -> pos -1
       "chr1\t4600\tid9\tN\t<INV>\t60\tPASS\tSVTYPE=INV;SVLEN=800;END=5400;SUPPORT=7"]
FILES = {
    "basic": HEAD + "\n".join(REC) + "\n",
    "no_format": "##fileformat=VCFv4.2\n#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\n" + "\n".join(REC[:3]) + "\n",
    "crlf": (HEAD + "\n".join(REC[:4]) + "\n").replace("\n", "\r\n"),
    "bad_blank": HEAD + REC[0] + "\n\n" + REC[1] + "\n",
    "bad_qual": HEAD + REC[0] + "\n" + REC[1].replace("\t.\t", "\t7.5\t") + "\n",
    "bad_info": HEAD + REC[0] + "\nchr1\t300\tx\tN\t<DEL>\t60\tPASS\tSVTYPE=DEL;SVLEN=-80=1\n",
    "bad_bnd": HEAD + "chr1\t300\tx\tN\t<BND>\t60\tPASS\tSVTYPE=BND\tGT\t0/1\n",
    "bnd_last_column": HEAD + "chr1\t300\tx\tN\t<BND>\t60\tPASS\tSVTYPE=BND\n",      # INFO keeps the newline: svtype "BND\n"
    "bad_columns": HEAD + "chr1\t300\tx\tN\t<DEL>\n",
}
GTS = [(0, 1, 30, 5, 6, ("1", 77)), (".", ".", 0, 0, 0, (None, None)), (0, 0, 0, 7, 0, (None, None)), (1, 1, 60, 0, 12, ("2", None))]

# block name: (reference call arguments, extra arguments of the genotype run, header with FORMAT lines, contig index whose first target is a BND)
BLOCKS = {
    "c1_ont_1mb": ([], [], False, None),
    "phased_phase": (["--phase"], ["--all-contigs"], True, 1),
    "c3_hifi_mosaic": (["--mosaic"], ["--contig", "ctg1"], True, None),      # ctg2 is not processed
    "hg008": ([], ["--all-contigs"], True, 2),
}


class Fatal(Exception):
    pass


def _patch_fatal():
    from sniffles import util
    import sniffles.vcf

    def fatal(msg):
        raise Fatal(msg)
    util.fatal_error = fatal
    sniffles.vcf.util.fatal_error = fatal


def _ref_config(*args):
    config = harness.make_config(*args)
    for k, v in STAMP.items():
        setattr(config, k, v)
    config.mode = "genotype_vcf"
    config.task_read_id_offset_mult = 10 ** 9
    return config


def make_parser_fixtures():
    from sniffles import vcf as rvcf
    config = _ref_config()
    expected = {"config": dict(STAMP), "files": {}}
    for name, text in FILES.items():
        path = os.path.join(OUT, name + ".vcf")
        with open(path, "w", newline="") as f:
            f.write(text)
        try:
            with open(path, "r") as f:
                v = rvcf.VCF(config, f)
                targets = list(v.read_svs_iter())
        except Fatal as e:
            expected["files"][name] = {"error": str(e)}
            continue
        out = io.StringIO()
        w = rvcf.VCF(config, out)
        w.rewrite_header_genotype(v.header_str)
        for i, t in enumerate(targets):
            t.genotype_match_sv, t.genotypes = None, {0: GTS[i % len(GTS)]}
            w.rewrite_genotype(t)
        expected["files"][name] = {
            "targets": [[t.contig, t.pos, t.svtype, t.svlen, t.end, t.bnd_info.mate_contig if t.bnd_info else None,
                         bool(t.bnd_info.is_first) if t.bnd_info else None, t.raw_vcf_line_index] for t in targets],
            "output": out.getvalue()}
    expected["genotypes"] = [list(g[:5]) + [list(g[5])] for g in GTS]
    expected["reference_defaults"] = {"genotype_format": config.genotype_format, "phase": bool(config.phase), "genotype_none": list(config.genotype_none[:5])}
    with open(os.path.join(OUT, "expected.json"), "w") as f:
        json.dump(expected, f, indent=1, sort_keys=True)


def load_block(name):
    """the record block of a fixture, as the call-path tests load it"""
    import test_oracle_golden as tog
    if name == "hg008":
        return tog._bam_block("hg008")
    return tog.load_fixture(name)[1]


def _target_lines(name, blk, cands_by_task, rng, bnd_first_task):
    """a target VCF's records derived from the block's own reference candidates, every edge case of the mode included"""
    lines = []
    add = lambda contig, pos1, ref, alt, info, fmt=True: lines.append(f"{contig}\t{pos1}\tt{len(lines)}\t{ref}\t{alt}\t.\tPASS\t{info}" + ("\tGT\t0/1" if fmt else ""))
    names = blk.contig_names
    for t in range(len(blk.task)):
        contig = names[int(blk.task[t]["contig"])]
        L = int(blk.task[t]["contig_len"])
        if t == bnd_first_task:                     # the task's first target is a BND: GenotypeTask raises UnboundLocalError
            add(contig, 3001, "N", f"N[{contig}:9000[", "SVTYPE=BND")
        cands = [c for c in cands_by_task[t] if not c["svtype"].startswith("SINGLE")]
        for k, c in enumerate(cands):
            sv, pos, svlen = c["svtype"], c["pos"], c["svlen"]
            if sv == "BND":
                alt = c["alt"]
                for d in (0, int(rng.integers(1, 200)), int(rng.integers(900, 1300))):
                    add(contig, pos + 1 + d, "N", alt, "SVTYPE=" + ("TRA" if k % 2 else "BND"))
                mate = alt.replace("]", "[").split("[")[1].split(":")[1]
                add(contig, pos + 1, "N", alt.replace(c["bnd"][0] + ":", "chrNotInHeader:").replace(":" + mate, ":" + mate), "SVTYPE=BND")
                continue
            lim = 250 * abs(svlen) ** 0.5
            for dp, dl in ((0, 0), (int(rng.integers(-20, 21)), int(rng.integers(-10, 11))), (int(rng.integers(-400, 401)), int(rng.integers(-200, 201))),
                           (int(lim) + int(rng.integers(1, 300)), 0), (int(rng.integers(1000, 3000)), 0)):
                add(contig, pos + 1 + dp, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN={svlen + (dl if svlen >= 0 else -dl)};END={pos + abs(svlen)}")
            if k % 5 == 0:
                add(contig, pos + 1, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN={svlen}")                            # exact duplicate
            if k % 7 == 0:
                add(contig, pos + 1, "N", f"<{sv}>", f"SVTYPE={sv}")                                          # no SVLEN: svlen -1 from REF / ALT
            if k % 11 == 0:
                add(contig, pos + 1, "N", "<CNV>", f"SVTYPE=CNV;SVLEN={svlen}")
            if k % 13 == 0:
                add(contig, pos + 1, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN=0")
            if k % 17 == 0:
                add(contig, pos + 1, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN={svlen}", fmt=False)                # SVTYPE keeps no newline: SVLEN last
            if k + 1 < len(cands) and cands[k + 1]["svtype"] == sv and abs(cands[k + 1]["svlen"]) == abs(svlen) and (cands[k + 1]["pos"] - pos) % 2 == 0:
                add(contig, (pos + cands[k + 1]["pos"]) // 2 + 1, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN={svlen}")   # equal distance to both
            b = pos // 5000 * 5000
            for off in (0, 499, 500, 4500, 4501, 4999):
                if k % 3 == 0:
                    add(contig, b + off + 1, "N", f"<{sv}>", f"SVTYPE={sv};SVLEN={svlen}")
        for pos1, alt, info in ((1, "<INS>", "SVTYPE=INS;SVLEN=400"), (0, "<DEL>", "SVTYPE=DEL;SVLEN=-300"), (5, "<DEL>", "SVTYPE=DEL;SVLEN=-2000000000"),
                                (L - 1, "<INS>", "SVTYPE=INS;SVLEN=80"), (L - 3, "<DUP>", "SVTYPE=DUP;SVLEN=5000"), (L, "<INS>", "SVTYPE=INS;SVLEN=80"),
                                (L + 50, "<DEL>", "SVTYPE=DEL;SVLEN=-90"), (400, "N[ctgNope:77[", "SVTYPE=BND"), (L // 2, "<CNV>", "SVTYPE=CNV;SVLEN=-7000")):
            add(contig, pos1, "N", alt, info)
    add("chrNotInBam", 5000, "N", "<DEL>", "SVTYPE=DEL;SVLEN=-500")
    return lines


def make_block_fixture(name):
    from sniffles import leadprov, parallel, util, vcf as rvcf
    from sniffles.region import Region
    call_args, extra, with_format, bnd_first = BLOCKS[name]
    blk = load_block(name)
    rng = np.random.default_rng(sum(map(ord, name)))
    cfg_call = harness.make_config(*call_args)
    cands = []
    for t in range(len(blk.task)):
        try:
            cands.append(harness.run_task(blk, t, cfg_call, finalize=False)["cands"])
        except UnboundLocalError:                 # a task whose first candidate is a BND fails in the reference's call path too
            cands.append([])
    head = ["##fileformat=VCFv4.2"] + [f"##contig=<ID={n},length={int(c['length'])}>" for n, c in zip(blk.contig_names, blk.contig)][:40]
    if with_format:
        head += ['##FORMAT=<ID=GT,Number=1,Type=String,Description="Genotype">', '##FORMAT=<ID=DR,Number=1,Type=Integer,Description="Number of reference reads">']
    head.append("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tSAMPLE")
    lines = _target_lines(name, blk, cands, rng, bnd_first)
    tpath = os.path.join(OUT, name + ".targets.vcf")
    with open(tpath, "w") as f:
        f.write("\n".join(head + lines) + "\n")
    config = _ref_config(*call_args, "--genotype-vcf", tpath, *extra)
    with open(tpath) as f:
        reader = rvcf.VCF(config, f)
        svs = list(reader.read_svs_iter())
    order = [s.raw_vcf_line_index for s in svs]
    by_contig = {}
    for s in svs:
        by_contig.setdefault(s.contig, []).append(s)
    task_of_contig = {blk.contig_names[int(blk.task[t]["contig"])]: t for t in range(len(blk.task))}
    out = io.StringIO()
    writer = rvcf.VCF(config, out)
    writer.rewrite_header_genotype(reader.header_str)
    task_id, failed, n_written = 0, [], 0
    for cname, c in zip(blk.contig_names, blk.contig):            # sniffles:313-358 with task_count_multiplier 0
        L = int(c["length"])
        if not util.should_process_contig(cname, L, config) or L - 1 <= 0:
            continue
        gsvs = [s for s in by_contig.get(cname, []) if 0 <= s.pos < L - 1]
        tid, task_id = task_id, task_id + 1
        if not gsvs:
            continue
        t = task_of_contig[cname]
        tr = None
        if int(blk.task[t]["tr_n"]) > 0:
            o, n = int(blk.task[t]["tr_off"]), int(blk.task[t]["tr_n"])
            tr = [(int(blk.tr[2 * (o + k)]), int(blk.tr[2 * (o + k) + 1])) for k in range(n)]
        tk = parallel.GenotypeTask(id=tid, sv_id=0, contig=cname, start=0, end=L - 1, config=config, tandem_repeats=tr, genotype_svs=gsvs)
        tk.lead_provider = leadprov.LeadProvider(config, tk.id * config.task_read_id_offset_mult, cname)
        tk.lead_provider.build_leadtab([Region(cname, 0, L - 1)], harness.DuckBam(blk, t))
        tk.build_leadtab = lambda tk=tk: ([], tk.lead_provider.read_count)
        try:
            res = tk.execute()
        except Exception as e:                    # parallel.py:747-752: the worker sends an ErrorResult, nothing is written
            failed.append([tid, cname, type(e).__name__])
            continue
        n_written += res.emit(vcf_out=writer, genotype_lineindex_order=order)
    with open(os.path.join(OUT, name + ".expected.json"), "w") as f:
        json.dump(dict(block=name, call_args=call_args, args=call_args + extra, stamp=STAMP, failed_tasks=failed, n_targets=len(svs),
                       n_written=n_written, output=out.getvalue()), f, indent=1)
    print(name, "targets", len(svs), "written", n_written, "failed", failed)


def main():
    harness.import_reference()
    _patch_fatal()
    os.makedirs(OUT, exist_ok=True)
    make_parser_fixtures()
    for name in (sys.argv[1:] or BLOCKS):
        make_block_fixture(name)


if __name__ == "__main__":
    main()
