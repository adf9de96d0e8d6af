"""SNF container (SURVEY 8f row 2) against a file the reference itself wrote (tests/golden/c2_ont_wgs_small.snf, made by
tests/golden/make_golden.py snf): the reader parses it, the candidates in it equal this package's candidates for the same block,
the 500-bp coverage entries equal the reshape-mean of the coverage, and the writer produces blocks that unpickle to the same content."""
import io
import json
import os

import numpy as np
import pytest

from oracle import genotype as ogt
from sniffles_b200 import abi, postprocess, snf, tasks
from sniffles_b200 import config as sconfig
import oracle.oracle as orc
import ref_fasta
from test_oracle_golden import GOLDEN, load_fixture

PATH = os.path.join(GOLDEN, "c2_ont_wgs_small.snf")
REF_SNF_COVERAGE = os.path.join(GOLDEN, "reference", "snf_coverage.json")
FIELDS = ["svtype", "pos", "end", "svlen", "support", "qual", "filter", "qc", "precise", "alt", "ref", "id", "fwd", "rev", "coverage_upstream", "coverage_start", "coverage_center",
          "coverage_end", "coverage_downstream", "genotypes", "rnames", "nm"]


def _numpy_cov_bins(blk, cfg, t, step, runs=None):
    """the SNF writer's bin means of task t's coverage vector, N runs `runs` zeroed (leadprov.py:470, snf.py:257-258)"""
    rec = blk.rec
    first = blk.cigar[rec["cigar_off"]]
    last = blk.cigar[rec["cigar_off"] + rec["n_cigar"] - 1]
    lead = np.where((first & 15) == 4, first >> 4, 0).astype(np.int64)
    trail = np.where(((last & 15) == 4) & (rec["n_cigar"] > 1), last >> 4, 0).astype(np.int64)
    alen = rec["l_seq"].astype(np.int64) - lead - trail
    tk = blk.task[rec["task"]]
    ok = (rec["mapq"] >= cfg.mapq) & ((rec["flag"] & 256) == 0) & (alen >= cfg.min_alignment_length) & (rec["pos"] >= tk["start"]) & (rec["pos"] < tk["end"])
    return ref_fasta.coverage_bins(ogt.coverage_vector(blk, ok, ogt.record_spans(blk), t, runs), step)


def snf_coverage_entries(bins, cfg, blocks):
    """the `_COVERAGE` dict SNFile.annotate_block_coverages stores in each SNF block at `blocks` (snf.py:260-264)"""
    step, bs = cfg.coverage_binsize_combine, cfg.snf_block_size
    per = bs // step
    return {b: {b + i * step: round(float(bins[b // bs * per + i])) for i in range(per) if b // bs * per + i < len(bins)} for b in blocks}


@pytest.mark.parametrize("name", sorted(ref_fasta.GOLDEN_FASTA))
def test_masked_bins_match_the_reference_snf_coverage(name):
    """The N-masked restatement of the writer's bin means equals the `_COVERAGE` the reference itself stored with --snf --reference
    (tests/golden/reference/snf_coverage.json, made by tests/golden/make_snf_coverage_golden.py), and the mask moves some of them."""
    with open(REF_SNF_COVERAGE) as f:
        gold = json.load(f)["blocks"][name]
    _, blk = load_fixture(name)
    text, seqs = ref_fasta.golden_fasta(name)
    assert ref_fasta.sha256(text) == gold["fasta_sha256"]
    cfg = sconfig.default_config("--snf", "x.snf", *gold["args"])
    runs = ref_fasta.task_runs(blk, seqs)
    moved = 0
    for t in range(len(blk.task)):
        contig = blk.contig_names[int(blk.task[t]["contig"])]
        want = {int(b): {int(p): v for p, v in e.items()} for b, e in gold["coverage"].get(contig, {}).items()}
        got = snf_coverage_entries(_numpy_cov_bins(blk, cfg, t, cfg.coverage_binsize_combine, runs.get(t)), cfg, want)
        assert got == want, (name, contig)
        plain = snf_coverage_entries(_numpy_cov_bins(blk, cfg, t, cfg.coverage_binsize_combine), cfg, want)
        moved += sum(got[b][p] != plain[b][p] for b in got for p in got[b])
    assert moved > 0 and sum(len(v) for v in gold["coverage"].values()) >= 5


def _our_candidates(fx, blk, cfg, res):
    """per task: the candidates as the SNF branch stores them (all of call_candidates' output, after finalize_candidates ran on them)"""
    out = []
    ranges = tasks.cand_ranges(res.cand, len(blk.task))
    for t in range(len(blk.task)):
        lo, hi = ranges[t]
        cfg.average_regional_nm = cfg.qc_nm_threshold = float(fx["tasks"][t]["mean_nm"])
        calls = postprocess.calls_from_result(res, t, lo, hi, blk.contig_names, blk.contig_names[int(blk.task[t]["contig"])], int(blk.task[t]["task_id"]), cfg, rec_nm=res.rec_nm, want_leads=True)
        postprocess.finalize_candidates(calls, True, cfg, float(res.task_cov_mean[t]))
        out.append(calls)
    return out


def test_reader_and_writer_against_the_reference_file():
    fx, blk = load_fixture("c2_ont_wgs_small")
    blk.mask = None                     # the reference file was written without --reference
    cfg = sconfig.default_config("--snf", "x.snf", *fx["args"])
    res = orc.run(blk, abi.Config.from_sniffles(cfg), 3, 2, keep_rec_nm=True)
    ours = _our_candidates(fx, blk, cfg, res)
    rd = snf.SNFReader(PATH)
    assert rd.header["snf_candidate_count"] == sum(len(c) for c in ours)
    assert sorted(rd.index) == sorted(blk.contig_names[int(t["contig"])] for t in blk.task if len(ours[int(t["task_id"])]))
    parts = []
    for t, calls in enumerate(ours):
        contig = blk.contig_names[int(blk.task[t]["contig"])]
        # ---- reader: every block of the reference file holds exactly our candidates of that window, field by field
        by_block = {}
        for c in calls:
            if c.svtype in snf.TYPES:
                by_block.setdefault(int(c.pos / cfg.snf_block_size) * cfg.snf_block_size, {}).setdefault(c.svtype, []).append(c)
        cov = _numpy_cov_bins(blk, cfg, t, cfg.coverage_binsize_combine)
        for block, types in by_block.items():
            ref_blocks = rd.read_blocks(contig, block)
            assert ref_blocks is not None and len(ref_blocks) == 1
            rb = ref_blocks[0]
            for svtype in snf.TYPES:
                mine, theirs = types.get(svtype, []), rb[svtype]
                assert len(mine) == len(theirs), (contig, block, svtype)
                for a, b in zip(mine, theirs):
                    for f in FIELDS:
                        assert getattr(snf.to_compat(a), f) == getattr(b, f), (contig, block, svtype, f, getattr(a, f, None), getattr(b, f))
                    assert {k: v for k, v in a.info.items() if v is not None} == {k: v for k, v in b.info.items() if v is not None}
            per_block = cfg.snf_block_size // cfg.coverage_binsize_combine
            want_cov = {block + i * cfg.coverage_binsize_combine: round(float(cov[block // cfg.snf_block_size * per_block + i])) for i in range(per_block) if block // cfg.snf_block_size * per_block + i < len(cov)}
            assert rb["_COVERAGE"] == want_cov
        # ---- writer: the same content through this package's writer
        buf = io.BytesIO()
        w = snf.SNFWriter(cfg, buf)
        for c in calls:
            w.store(c)
        w.annotate_block_coverages(cov)
        w.write_and_index()
        parts.append((int(blk.task[t]["task_id"]), contig, dict(w.index), buf.getvalue(), len(calls), float(res.task_cov_mean[t])))
    out = io.BytesIO()
    n = snf.write_results(out, cfg, parts, list(blk.contig_names))
    assert n == rd.header["snf_candidate_count"]
    tmp = PATH + ".roundtrip.tmp"
    with open(tmp, "wb") as f:
        f.write(out.getvalue())
    try:
        mine = snf.SNFReader(tmp)
        assert {c: {b: len(v) for b, v in d.items()} for c, d in mine.index.items()} == {c: {b: len(v) for b, v in d.items()} for c, d in rd.index.items()}
        a, b = list(mine.all_calls()), list(rd.all_calls())
        assert len(a) == len(b) == sum(1 for calls in ours for c in calls if c.svtype in snf.TYPES)
        for (c1, b1, x), (c2, b2, y) in zip(a, b):
            assert (c1, b1) == (c2, b2) and all(getattr(x, f) == getattr(y, f) for f in FIELDS)
            assert type(x).__module__ == "sniffles.sv" and type(x).__name__ == "SVCall"
        mine.close()
    finally:
        os.remove(tmp)
    rd.close()
