"""Generates tests/golden/regions/expected.json: the unmodified reference's whole-sample run with --regions / --region (sniffles:131-590,
config.py:482-505, LeadProvider.build_leadtab over the task's regions, leadprov.py:445-470) on the cases of tests/regions_common.py.  Runs
only where the reference's source tree exists (oracle/pyref/harness.py finds it, behind its stub pysam); the fixture travels, the
reference does not.

    python tests/golden/make_regions_golden.py

As tests/golden/make_call_sample_golden.py, except that each task's lead provider reads the task's regions (config.regions_by_contig,
parsed by the reference's own SnifflesConfig) through a DuckBam over all of the contig's records, whose fetch applies the overlap test of
bam.fetch and refuses start < 0 or start > end with ValueError as pysam's parse_region does (restated, not pinned)."""
import io
import json
import logging
import math
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests"), HERE]
logging.disable(logging.CRITICAL)

import call_sample_common as csc  # noqa: E402
import harness  # noqa: E402
import regions_common as rc  # noqa: E402
from make_reference_golden import TextFasta  # noqa: E402
from sniffles_b200 import bamio  # noqa: E402


class RegionBam(harness.DuckBam):
    def fetch(self, contig, start, end, until_eof=False):
        if start < 0:
            raise ValueError(f"start out of range ({start})")
        if start > end:
            raise ValueError(f"invalid coordinates: start ({start}) > stop ({end})")
        for i in self.idx:
            rd = harness.DuckRead(self.block, int(i))
            if rd.reference_start < end and rd.reference_start + max(rd.reference_end - rd.reference_start, 1) > start:
                yield rd


def reference_run(case, tmp):
    from sniffles import leadprov, parallel, snf as refsnf, util, vcf as refvcf
    from sniffles.region import Region
    import pysam
    name = rc.CASES[case][0]
    paths = csc.write_inputs(name, os.path.join(tmp, name))
    bam = bamio.BamFile(paths["bam"])
    vcf_path, snf_path = os.path.join(tmp, case + ".vcf"), os.path.join(tmp, case + ".snf")
    args = rc.case_args(case, paths, bam, tmp, vcf_path, snf_path)[4:]
    config = harness.make_config(*args)
    for k, v in csc.STAMP.items():
        setattr(config, k, v)
    config.mode, config.input = "call_sample", paths["bam"]
    config.sample_ids_vcf = [(0, "SAMPLE" if config.sample_id is None else config.sample_id)]
    total_mapped = sum(bam.count_mapped(n) or 0 for n, _ in bam.contigs)
    config.task_read_id_offset_mult = 10 ** 9 if total_mapped == 0 else 10 ** math.ceil(math.log(total_mapped) + 1)
    trs = util.load_tandem_repeats(config.tandem_repeats, config.tandem_repeat_region_pad) if config.tandem_repeats else {}
    contigs, contig_lengths, planned = [], [], []
    for cname, L in bam.contigs:
        if not util.should_process_contig(cname, L, config):
            continue
        contigs.append(cname)
        contig_lengths.append((cname, L))
        start = 0
        while start < L - 1:
            planned.append((len(planned), cname, start, min(L - 1, start + L)))
            start += L
    config.contig_lengths = contig_lengths
    pysam.FastaFile = TextFasta
    out = io.StringIO()
    writer = refvcf.VCF(config, out)
    writer.open_reference()
    writer.write_header(contig_lengths)
    snf_out = refsnf.SNFile(config, open(snf_path, "wb")) if config.snf else None
    results, failed = [], []
    for tid, cname, s, e in planned:
        cidx = bam.name_to_id[cname]
        L = bam.get_reference_length(cname)
        blk = bamio.pack_records(bam.contigs, [(0, r) for r in bam.fetch(cname, 0, L)], [(cidx, 0, L, tid)])
        regions = config.regions_by_contig.get(cname)
        tk = parallel.CallTask(id=tid, sv_id=0, contig=cname, start=s, end=e, config=config, assigned_process_id=None,
                               tandem_repeats=trs.get(cname), genotype_svs=None, regions=regions)
        try:
            tk.lead_provider = leadprov.LeadProvider(config, tid * config.task_read_id_offset_mult, cname)
            tk.lead_provider.build_leadtab(regions if regions else [Region(cname, s, e)], RegionBam(blk, 0))
            tk.build_leadtab = lambda tk=tk: ([], tk.lead_provider.read_count)
            results.append(tk.execute())
        except Exception as ex:                 # parallel.py:747-752: the worker sends an ErrorResult, nothing is written
            failed.append([tid, cname, type(ex).__name__])
    results.sort(key=lambda r: r.task_id)
    for r in results:
        r.emit(vcf_out=writer, snf_out=snf_out)
    got = {"input": name, "args": [a if not a.startswith(tmp) else os.path.basename(a) for a in args],
           "regions_by_contig": {c: [[r.start, r.end] for r in v] for c, v in config.regions_by_contig.items()},
           "failed_tasks": failed, "n_tasks": len(planned), "n_written": writer.call_count, "vcf": csc.vcf_digest(out.getvalue())}
    if snf_out is not None:
        snf_out.write_results(config, contigs)
        snf_out.close()
        got["snf"] = csc.snf_digest(snf_path)
    bam.close()
    return got


def reference_genotype(case, tmp):
    """GenotypeTask.execute (parallel.py:300-369) per planned task with the task's regions, written by GenotypeResult.emit in task order"""
    from sniffles import leadprov, parallel, util, vcf as rvcf
    from sniffles.region import Region
    name, _, _, targets = rc.GENOTYPE_CASES[case]
    paths = csc.write_inputs(name, os.path.join(tmp, name))
    bam = bamio.BamFile(paths["bam"])
    tpath = os.path.join(HERE, "genotype", targets)
    args = rc.case_args(case, paths, bam, tmp, os.path.join(tmp, case + ".vcf"), None, rc.GENOTYPE_CASES)[4:] + ["--genotype-vcf", tpath]
    config = harness.make_config(*args)
    for k, v in csc.STAMP.items():
        setattr(config, k, v)
    config.mode, config.task_read_id_offset_mult = "genotype_vcf", 10 ** 9
    with open(tpath) as f:
        reader = rvcf.VCF(config, f)
        svs = list(reader.read_svs_iter())
    order = [s.raw_vcf_line_index for s in svs]
    by_contig = {}
    for sv in svs:
        by_contig.setdefault(sv.contig, []).append(sv)
    out = io.StringIO()
    writer = rvcf.VCF(config, out)
    writer.rewrite_header_genotype(reader.header_str)
    task_id, failed, n_written = 0, [], 0
    for cname, L in bam.contigs:
        if not util.should_process_contig(cname, L, config) or L - 1 <= 0:
            continue
        gsvs = [sv for sv in by_contig.get(cname, []) if 0 <= sv.pos < L - 1]
        tid, task_id = task_id, task_id + 1
        if not gsvs:
            continue
        regions = config.regions_by_contig.get(cname)
        blk = bamio.pack_records(bam.contigs, [(0, r) for r in bam.fetch(cname, 0, L)], [(bam.name_to_id[cname], 0, L, tid)])
        tk = parallel.GenotypeTask(id=tid, sv_id=0, contig=cname, start=0, end=L - 1, config=config, genotype_svs=gsvs, regions=regions)
        try:
            tk.lead_provider = leadprov.LeadProvider(config, tk.id * config.task_read_id_offset_mult, cname)
            tk.lead_provider.build_leadtab(regions if regions else [Region(cname, 0, L - 1)], RegionBam(blk, 0))
            tk.build_leadtab = lambda tk=tk: ([], tk.lead_provider.read_count)
            res = tk.execute()
        except Exception as e:                    # parallel.py:747-752: the worker sends an ErrorResult, nothing is written
            failed.append([tid, cname, type(e).__name__])
            continue
        n_written += res.emit(vcf_out=writer, genotype_lineindex_order=order)
    bam.close()
    return {"input": name, "targets": targets, "regions_by_contig": {c: [[r.start, r.end] for r in v] for c, v in config.regions_by_contig.items()},
            "failed_tasks": failed, "n_targets": len(svs), "n_written": n_written, "output": out.getvalue()}


def parser_cases():
    """the reference's config parsing of the inputs of its own src/tests/test_regions.py, plus the --region strings"""
    from unittest.mock import patch, mock_open
    from sniffles.config import SnifflesConfig
    out = {}
    inputs = {"good_file": "\n# comment line is ok\nchr1\t100\t200\n\nchr1\t500\t600\n\nchr3\t500\t600\n\n        ",
              "invalid_lines": "\n... <- invalid line\nchr1\t100\t200\n  valid line\n\n",
              "unsorted_overlap": "chr2\t500\t900\nchr1\t10\t20\nchr2\t100\t600\nchr2\t100\t600\nchr1\t5\t6 extra\tfields\n"}
    for k, data in inputs.items():
        with patch("builtins.open", mock_open(read_data=data)):
            cfg = SnifflesConfig("--input", "input.bam", "--vcf", "out.vcf", "--regions", "regions.bed")
        out[k] = {"bed": data, "regions_by_contig": {c: [[r.contig, r.start, r.end] for r in v] for c, v in cfg.regions_by_contig.items()}}
    strings = ["chr1:100-200", "chr1:5-", "chr2:7-9", "bad", "chr1:1-2:3", "chr1:300-250"]
    cfg = SnifflesConfig("--input", "input.bam", "--vcf", "out.vcf", *[x for s in strings for x in ("--region", s)])
    out["region_strings"] = {"strings": strings, "regions_by_contig": {c: [[r.contig, r.start, r.end] for r in v] for c, v in cfg.regions_by_contig.items()}}
    return out


def main():
    harness.import_reference()
    tmp = tempfile.mkdtemp()
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", "stamp": csc.STAMP, "parser": parser_cases(), "cases": {}}
    for case in rc.CASES:
        got = out["cases"][case] = reference_run(case, tmp)
        print(case, "tasks", got["n_tasks"], "records", len(got["vcf"]["records"]), "failed", got["failed_tasks"],
              "snf candidates", got.get("snf", {}).get("snf_candidate_count"), flush=True)
    out["genotype"] = {}
    for case in rc.GENOTYPE_CASES:
        got = out["genotype"][case] = reference_genotype(case, tmp)
        print(case, "targets", got["n_targets"], "written", got["n_written"], "failed", got["failed_tasks"], flush=True)
    os.makedirs(os.path.dirname(rc.EXPECTED), exist_ok=True)
    with open(rc.EXPECTED, "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
