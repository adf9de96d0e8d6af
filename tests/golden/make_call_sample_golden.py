"""Generates tests/golden/call_sample/expected.json: the unmodified reference's whole-sample run (`sniffles -i sample.bam -v out.vcf
[--snf out.snf]`, sniffles:131-590) on the inputs and argument sets of tests/call_sample_common.py.  Runs only where the reference's
source tree exists (oracle/pyref/harness.py finds it, behind its stub pysam); the fixture travels, the reference does not.

    python tests/golden/make_call_sample_golden.py

Per case: the reference's planning (util.should_process_contig over the BAM header, one task per processed contig as task_count_multiplier
0 plans it, util.load_tandem_repeats), config.task_read_id_offset_mult by the rule of sniffles:304-309 from the index's mapped-read counts,
every planned task through the reference's CallTask.execute (its lead provider built from the task's records, read by this package's
host BAM reader and exposed through oracle/pyref's DuckBam), the results emitted in task-id order into the reference's VCF.write_header /
write_call and SNFile.write_results.  `command`, `fileDate` and the version are fixed (call_sample_common.STAMP)."""
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
from make_reference_golden import TextFasta  # noqa: E402
from sniffles_b200 import bamio  # noqa: E402


def reference_run(case, tmp):
    from sniffles import leadprov, parallel, snf as refsnf, util, vcf as refvcf
    from sniffles.region import Region
    import pysam
    name, _ = csc.CASES[case]
    paths = csc.write_inputs(name, os.path.join(tmp, name))
    vcf_path, snf_path = os.path.join(tmp, case + ".vcf"), os.path.join(tmp, case + ".snf")
    args = csc.case_args(case, paths, vcf_path, snf_path)[4:]
    config = harness.make_config(*args)
    for k, v in csc.STAMP.items():
        setattr(config, k, v)
    config.mode, config.input = "call_sample", paths["bam"]
    config.sample_ids_vcf = [(0, "SAMPLE" if config.sample_id is None else config.sample_id)]
    bam = bamio.BamFile(paths["bam"])
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
        while start < L - 1:                    # task_count 1: task_length = L
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
        blk = bamio.pack_records(bam.contigs, [(0, r) for r in bam.fetch(cname, s, e)], [(cidx, s, e, tid)])
        tk = parallel.CallTask(id=tid, sv_id=0, contig=cname, start=s, end=e, config=config, assigned_process_id=None,
                               tandem_repeats=trs.get(cname), genotype_svs=None, regions=None)
        tk.lead_provider = leadprov.LeadProvider(config, tid * config.task_read_id_offset_mult, cname)
        tk.lead_provider.build_leadtab([Region(cname, s, e)], harness.DuckBam(blk, 0))
        tk.build_leadtab = lambda tk=tk: ([], tk.lead_provider.read_count)
        try:
            results.append(tk.execute())
        except Exception as ex:                 # parallel.py:747-752: the worker sends an ErrorResult, nothing is written
            failed.append([tid, cname, type(ex).__name__])
    results.sort(key=lambda r: r.task_id)
    for r in results:
        r.emit(vcf_out=writer, snf_out=snf_out)
    got = {"input": name, "args": csc.CASES[case][1], "failed_tasks": failed, "n_tasks": len(planned),
           "task_read_id_offset_mult": config.task_read_id_offset_mult, "n_written": writer.call_count, "vcf": csc.vcf_digest(out.getvalue())}
    if snf_out is not None:
        snf_out.write_results(config, contigs)
        snf_out.close()
        got["snf"] = csc.snf_digest(snf_path)
    bam.close()
    return got


def main():
    harness.import_reference()
    tmp = tempfile.mkdtemp()
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", "stamp": csc.STAMP, "cases": {}}
    for case in csc.CASES:
        got = out["cases"][case] = reference_run(case, tmp)
        print(case, "tasks", got["n_tasks"], "records", len(got["vcf"]["records"]), "failed", got["failed_tasks"],
              "snf candidates", got.get("snf", {}).get("snf_candidate_count"), flush=True)
    # combine mode over two samples' SNFs (the reference's own files of two cases): CombineTask per contig, as harness.reference_combine runs it
    snfs = [os.path.join(tmp, case + ".snf") for case in csc.COMBINE_CASES]
    contigs = [(n, int(c["length"])) for n, c in zip(csc.load_block("phased_phase").contig_names, csc.load_block("phased_phase").contig)]
    _, calls, _ = harness.reference_combine(snfs, contigs)
    out["combine"] = {name: csc.combine_digest(calls[name]) for name, _ in contigs}
    print("combine", {k: len(v) for k, v in out["combine"].items()}, flush=True)
    os.makedirs(os.path.dirname(csc.EXPECTED), exist_ok=True)
    with open(csc.EXPECTED, "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
