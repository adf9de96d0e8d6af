"""Generates tests/golden/rnames/: the unmodified reference's whole-sample runs with --output-rnames on the cases of
tests/rnames_common.py, through make_call_sample_golden.reference_run (the same planning, tasks and writers as tests/golden/call_sample/),
stored in rnames_common's forms; the reference-written SNFs of rnames_common.COMBINE_CASES as data fixtures; and the reference's combine
(harness.reference_combine with --output-rnames) over those two files.  Runs only where the reference's source tree exists.

    python tests/golden/make_rnames_golden.py"""
import json
import os
import shutil
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests"), HERE]

import call_sample_common as csc  # noqa: E402
import make_call_sample_golden as mcs  # noqa: E402
import rnames_common as rnc  # noqa: E402
import harness  # noqa: E402


def main():
    harness.import_reference()
    rnc.register()
    csc.vcf_digest, csc.snf_digest = rnc.vcf_form, rnc.snf_form       # reference_run stores this fixture's forms
    tmp = tempfile.mkdtemp()
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", "stamp": csc.STAMP, "cases": {}}
    for case in rnc.CASES:
        got = out["cases"][case] = mcs.reference_run(case, tmp)
        names = sum(len(r[-1] or []) for r in got["vcf"]["records"])
        print(case, "records", len(got["vcf"]["records"]), "names", names, "snf candidates", got.get("snf", {}).get("snf_candidate_count"), flush=True)
    os.makedirs(rnc.GOLDEN, exist_ok=True)
    snfs = []
    for case in rnc.COMBINE_CASES:
        snfs.append(os.path.join(rnc.GOLDEN, case + ".snf"))
        shutil.copyfile(os.path.join(tmp, case + ".snf"), snfs[-1])
    blk = csc.load_block("phased_phase")
    contigs = [(n, int(c["length"])) for n, c in zip(blk.contig_names, blk.contig)]
    _, _, lines = harness.reference_combine(snfs, contigs, config_args=("--output-rnames",))
    out["combine"] = {"contigs": contigs, "records": rnc.combine_form(lines)}
    print("combine records", len(lines), flush=True)
    with open(rnc.EXPECTED, "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
