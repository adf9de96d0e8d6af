"""--output-rnames without a GPU: the snfb_rnames_view layout, the host decode of the device's names text into per-candidate lists, the
RNAMES entry and the pickled SNF candidate with and without the option, and combine mode's RNAMES against the reference's combine of two
SNFs that carry names (tests/golden/rnames/, written by tests/golden/make_rnames_golden.py), through the grouping restatement."""
import ctypes as C
import gzip
import io
import json
import os
import pickle
import sys

import numpy as np

import rnames_common as rnc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "pyref"))
from oracle import combine as ocombine                             # noqa: E402
from sniffles_b200 import abi, binding, combine, postprocess, snf, vcf   # noqa: E402
from sniffles_b200 import config as sconfig                         # noqa: E402

with open(rnc.EXPECTED) as _f:
    GOLD = json.load(_f)


def test_rnames_view_layout_matches_the_library():
    assert binding.lib().snfb_sizeof(18) == C.sizeof(abi.RnamesView) == 40


def _names(names):
    text = b"".join(names)
    off = np.zeros(len(names) + 1, "<u4")
    off[1:] = np.cumsum([len(n) for n in names])
    return binding.ReadNames(np.frombuffer(text, "u1").copy(), off)


def test_decode_per_candidate():
    long_name = bytes(ord("A") + k % 26 for k in range(254))
    names = [b"r", b"read/2", long_name, b"m64011_190830_220126/1/ccs", b"x,y"]
    rn = _names(names)
    rn_off = np.array([0, 0, 1, 3, 3, 5], "<u4")                  # five candidates: an empty one first, an empty one in the middle
    got = rn.per_candidate(rn_off, 0, 5)
    assert got == [[], ["r"], ["read/2", long_name.decode()], [], ["m64011_190830_220126/1/ccs", "x,y"]]
    assert all(type(s) is str for c in got for s in c)
    assert rn.per_candidate(rn_off, 2, 4) == got[2:4]
    assert rn.per_candidate(rn_off, 3, 3) == []
    assert _names([]).per_candidate(np.zeros(1, "<u4"), 0, 0) == []


def _call(rnames):
    return postprocess.SVCall(contig="ctg1", pos=1000, id="INS.0S0", ref="N", alt="<INS>", qual=60, filter="PASS", info={"STDEV_POS": 0},
                              svtype="INS", svlen=120, end=1001, genotypes={0: (0, 1, 20, 3, 2, (None, None))}, precise=True, support=2,
                              rnames=rnames, qc=True, nm=-1.0, postprocess=None, fwd=1, rev=1)


def _vcf_line(args, call):
    cfg = sconfig.default_config(*args)
    cfg.sample_ids_vcf = [(0, "SAMPLE")]
    buf = io.StringIO()
    vcf.VCFWriter(cfg, buf).write_call(call)
    return buf.getvalue().rstrip("\n")


def _snf_candidates(args, call):
    cfg = sconfig.default_config("--snf", "x.snf", *args)
    buf = io.BytesIO()
    w = snf.SNFWriter(cfg, buf)
    w.store(call)
    w.write_and_index()
    return pickle.loads(gzip.decompress(buf.getvalue()))["INS"]


def test_vcf_and_snf_with_and_without_the_option():
    names = ["b9d3-1", "a0f1-2"]
    with_names = _vcf_line(["--output-rnames"], _call(list(names)))
    without = _vcf_line([], _call(list(names)))
    assert ";SUPPORT=2;RNAMES=b9d3-1,a0f1-2;COVERAGE=" in with_names
    assert "RNAMES" not in without
    assert rnc.split_rnames(with_names) == (without, names)
    assert _vcf_line([], _call(None)) == without                  # a call built without names: the output the option leaves alone
    (c,) = _snf_candidates(["--output-rnames"], _call(list(names)))
    assert type(c.rnames) is list and c.rnames == names and all(type(s) is str for s in c.rnames)
    (c,) = _snf_candidates([], _call(list(names)))
    assert c.rnames is None


def _combine_calls():
    cfg = sconfig.default_config("--output-rnames")
    cfg.mode = "combine"
    cfg.snf_input_info, cfg.sample_ids_vcf = [], []
    for k, case in enumerate(rnc.COMBINE_CASES):
        path = os.path.join(rnc.GOLDEN, case + ".snf")
        r = snf.SNFReader(path)
        sid = r.header["config"].get("sample_id") or case
        r.close()
        cfg.snf_input_info.append({"internal_id": k, "sample_id": sid, "filename": path})
        cfg.sample_ids_vcf.append((k, sid))
    readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in cfg.snf_input_info}
    calls = []
    try:
        for tid, (name, length) in enumerate(GOLD["combine"]["contigs"]):
            task = combine.CombineTask(tid, name, 0, length - 1, cfg)
            plan = combine.Plan()
            task.plan(readers, plan)
            calls += combine.CombineTask.emit([task], plan, ocombine.combine_groups(combine.plan_arrays(plan, cfg), cfg))[0]
    finally:
        for r in readers.values():
            r.close()
    return cfg, calls


def test_combine_rnames_equal_the_reference_in_order():
    from harness import FakeFasta
    cfg, calls = _combine_calls()
    buf = io.StringIO()
    w = vcf.VCFWriter(cfg, buf, reference=FakeFasta())
    for c in calls:
        w.write_call(c)
    got = rnc.combine_form(buf.getvalue().splitlines())
    want = GOLD["combine"]["records"]
    assert len(got) == len(want) > 0
    assert got == want
    # the names are the SNFs' own lists, concatenated over the group's candidates: some records merge both samples
    assert any(len(r[4]) > len(set(r[4])) for r in want)
