"""Generates tests/golden/consensus/expected.json: the unmodified reference (oracle/pyref/harness.run_task, --no-qc so every call survives)
on every case block of tests/consensus_common.py, with what shows that each case reaches its edge.  Runs only where the reference's
source tree exists.

    python tests/golden/make_consensus_golden.py

Per case: the block digest, the CLI args, every call's type, position, length and ALT (as its length and SHA-256 prefix), and one entry
per consensus the reference built (consensus.novel_from_reads wrapped to log its inputs: L, skip, the number of other reads, the
best read's name and, for fewer than 8 other reads, every read's name, length and start; and util.most_common wrapped to log every
voted column: its aligned rows nal = len(nums) - 1, the top two counts, and whether the winner replaced the best read's base).  Both wrappers return what they wrap unchanged."""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests")]

import consensus_common as cc  # noqa: E402
import harness  # noqa: E402

OUT = os.path.join(HERE, "consensus", "expected.json")


def main():
    harness.import_reference()
    from sniffles import consensus, util
    log, inside = [], []
    most_common, novel_from_reads = util.most_common, consensus.novel_from_reads

    def logged_most_common(nums):
        if not inside:                     # phase_sv calls it too
            return most_common(nums)
        nums = list(nums)
        top = most_common(nums)
        t1 = top[1][0] if len(top) > 1 else 0
        changed = len(top) > 1 and top[0][0] - top[1][0] >= 3 and top[0][1] != nums[0]
        v = log[-1]["votes"]
        key = f"{len(nums) - 1},{top[0][0]},{t1},{int(changed)}"
        v[key] = v.get(key, 0) + 1
        return top

    def logged_novel_from_reads(best_lead, other_leads, klen, skip, skip_repetitive, debug=False):
        e = dict(L=len(best_lead.seq), skip=skip, n_other=len(other_leads), best=best_lead.read_qname, votes={})
        if len(other_leads) < 8:          # the reads' (name, length, start): what the best-read choice is checked on
            e["leads"] = [[ld.read_qname, len(ld.seq), ld.ref_start] for ld in [best_lead] + list(other_leads)]
        log.append(e)
        inside.append(1)
        try:
            return novel_from_reads(best_lead, other_leads, klen, skip, skip_repetitive, debug)
        finally:
            inside.pop()

    util.most_common, consensus.novel_from_reads = logged_most_common, logged_novel_from_reads
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", "cases": {}}
    for name in cc.CASES:
        blk, metas, args = cc.build(name)
        del log[:]
        got = harness.run_task(blk, 0, harness.make_config(*args))
        calls = [[c["svtype"], c["pos"], c["svlen"], len(c["alt"]), cc.alt_digest(c["alt"])] for c in got["final"]]
        out["cases"][name] = dict(digest=cc.digest(blk), args=list(args), calls=calls, consensus=[dict(x) for x in log])
        print(name, "calls", len(calls), "consensus", [(x["L"], x["skip"], x["n_other"]) for x in log], flush=True)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    with open(OUT, "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
