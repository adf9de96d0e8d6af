"""Generates tests/golden/combine_reference/expected.json: the whole VCF the UNMODIFIED reference's combine mode writes with `--reference`
for the cases of tests/combine_reference_common.py, over combine_cli_common's SNF inputs and the seeded FASTA of combine_reference_common.

The reference runs as make_population_golden runs it (the setup of sniffles:371-481 restated, each task with a pickled copy of the
config, its CombineTask, CombineResult / CombineResultTmpFile and VCF writer), with the main writer's reference opened as sniffles:253-256
opens it.  The stub `pysam.FastaFile` is replaced by make_reference_golden's reader of the FASTA text, so VCF.write_call and the
CombineResultTmpFile parts (result.py:210-214) read the real sequence.  Stored per case: the VCF in combine_cli_common's compact form
(run-stamp lines left out), the calls CombineResultTmpFile set aside, and the records counted by how their alleles were resolved.
Run where the reference's source tree is available (oracle/pyref/harness.py finds it):
    python tests/golden/make_combine_reference_golden.py"""
import io
import json
import logging
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests"), HERE]
logging.disable(logging.CRITICAL)

import combine_cli_common as ccc                   # noqa: E402
import combine_reference_common as crc             # noqa: E402
import harness                                     # noqa: E402
import make_population_golden as mpg               # noqa: E402
import population_common as pc                     # noqa: E402
from make_reference_golden import TextFasta        # noqa: E402


def reference_vcf(files, extra, fasta, population, tmp):
    """the reference's combine VCF text with --reference `fasta` (and --combine-population), and the calls it set aside"""
    from sniffles import vcf as refvcf
    args = [*extra, "--reference", fasta] + (["--combine-population", pc.snf_path(population)] if population else [])
    config, contig_lengths, tasks, result_class = mpg._setup(files, args, tmp)
    buf = io.StringIO()
    vcf_out = refvcf.VCF(config, buf)
    vcf_out.open_reference()                         # sniffles:253-256
    vcf_out.write_header(contig_lengths)
    unsorted = 0
    for t in tasks:
        t.result = t.execute()
        if result_class is not None and os.path.exists(t.result.tmpfile_unsorted):
            with open(t.result.tmpfile_unsorted) as f:
                unsorted += sum(1 for _ in f)
            os.unlink(t.result.tmpfile_unsorted)
        t.result.emit(vcf_out=vcf_out)
    return buf.getvalue(), unsorted


def main():
    harness.import_reference()
    import pysam
    pysam.FastaFile = TextFasta
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via tests/golden/make_combine_reference_golden.py", "fasta_sha256": {},
           "headers": [], "records": [], "cases": {}}
    pools = {"headers": {}, "records": {}}

    def index(kind, item):
        key = json.dumps(item)
        if key not in pools[kind]:
            pools[kind][key] = len(out[kind])
            out[kind].append(item)
        return pools[kind][key]
    with tempfile.TemporaryDirectory() as tmp:
        fa_dir = os.path.join(tmp, "fasta")
        os.makedirs(fa_dir)
        fastas = {}
        for kind in ("full", "no_ctg2"):
            fastas[kind], out["fasta_sha256"][kind] = crc.fasta_files(kind, fa_dir)
        os.chdir(ccc.write_inputs(os.path.join(tmp, "in")))
        for label, files, extra, kind, population in crc.CASES:
            d = os.path.join(tmp, label)
            os.makedirs(d)
            text, unsorted = reference_vcf(files, extra, fastas[kind], population, d)
            lines = ccc.vcf_lines(text)
            out["cases"][label] = {"inputs": files, "args": extra, "fasta": kind, "population": population, "dropped": unsorted,
                                   "alleles": crc.allele_counts(text),
                                   "headers": [index("headers", x) for x in lines if isinstance(x, str)],
                                   "records": [index("records", x) for x in lines if not isinstance(x, str)]}
            print(label, "records", sum(not isinstance(x, str) for x in lines), "dropped", unsorted, crc.allele_counts(text), flush=True)
    os.makedirs(os.path.dirname(crc.EXPECTED), exist_ok=True)
    with open(crc.EXPECTED, "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
