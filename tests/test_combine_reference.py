"""Combine mode with `--reference`, without a GPU: the device context, the chunk plan and the grouping are stood in for, so that the
driver's use of the reference is pinned on its own.  The reference is a duck-typed `Reference` over sequences held in memory; the
calls of each task are made by hand.

  * the contigs handed to tasks.reference_for follow --contig / --regions, and the load is logged as sniffles:255 logs it;
  * the writer of the CombineResultTmpFile ordering gets the reference;
  * Reference.prefetch is called once per pass, with vcf.reference_intervals of exactly the calls that pass writes;
  * a FASTA that cannot be opened leaves the output equal to a run without --reference, plus one error line."""
import gzip
import logging

import numpy as np
import pytest

import combine_cli_common as ccc
from sniffles_b200 import combine, combine_run, postprocess, tasks, vcf
from sniffles_b200 import config as sconfig

S4 = ["s1.snf", "s2.snf", "s3.snf", "s4.snf"]


class DuckReference:
    """pysam.FastaFile look-alike with prefetch: every prefetch call's intervals are kept"""

    def __init__(self, seqs):
        self.seqs, self.prefetched = seqs, []

    def fetch(self, contig, start=None, end=None):
        s = self.seqs[contig]
        start = 0 if start is None else start
        end = len(s) if end is None else end
        if start < 0 or start > end:
            raise ValueError("invalid coordinates")
        return s[start:min(end, len(s))]

    def prefetch(self, intervals):
        self.prefetched.append(list(intervals))
        return sum(e - s for _, s, e in intervals)


class FakeContext:
    """snfb_combine_plan's result shape with every candidate kept and no chains: the calls come from `hand_made_batches`"""

    def combine_plan(self, flat, config):
        n = len(flat["pos"])
        return dict(perm=np.arange(n, dtype="<u4"), chains=np.zeros((0, 6), "<u4"), chunks=np.zeros((0, 6), "<i4"),
                    cand_group=np.zeros(n, "<u4"), emit_chunk=np.full(n, -1, "<i4"), emit_ord=np.zeros(n, "<u4"),
                    cov_non=np.zeros((n, flat["n_samples"]), "<i4"))


def _call(task, svtype, pos, svlen, alt):
    gt = {0: (0, 1, 20, 5, 5, (None, None), f"{svtype}.0"), 1: (0, 0, 20, 9, 0, (None, None), "NULL")}
    return postprocess.SVCall(contig=task.contig, pos=pos, id=f"{svtype}.{pos:X}M{task.id:X}", ref="N", alt=alt, qual=30, filter="PASS", info={},
                              svtype=svtype, svlen=svlen, end=pos + abs(svlen), genotypes=gt, precise=True, support=5, rnames=None, qc=True,
                              nm=-1, postprocess=None, fwd=3, rev=2, coverage_upstream=20, coverage_start=20, coverage_center=20,
                              coverage_end=20, coverage_downstream=20)


@pytest.fixture
def run(monkeypatch, tmp_path):
    """patches the device context, tasks.reference_for and the grouping; returns (run(args, budget) -> (stats, VCF text), log of the
    reference_for calls, the calls made per pass)"""
    inputs = ccc.write_inputs(str(tmp_path / "in"))
    monkeypatch.chdir(inputs)
    ctx = FakeContext()
    monkeypatch.setattr(tasks, "device_context", lambda device=0: ctx)
    passes = []

    def hand_made_batches(task_list, plan, out):
        made = []
        result = {}
        for k, t in enumerate(task_list):
            b = t.block_indices[0]
            calls = [_call(t, "DEL", b + 1_000, -150, "<DEL>"), _call(t, "INS", b + 2_000, 60, "ACGT" * 15), _call(t, "DUP", b + 3_000, 400, "<DUP>")]
            made.extend(calls)
            result[k] = [(0, c) for c in calls]
        passes.append((made, vcf.reference_intervals(made, task_list[0].config)))
        return result
    monkeypatch.setattr(combine.CombineTask, "emit_batches", staticmethod(hand_made_batches))

    def go(args, budget=None, name="out.vcf"):
        cfg = sconfig.SnifflesConfig("-i", *args[0], "-v", str(tmp_path / name), *args[1])
        st = {}
        combine_run.combine_snfs(cfg, budget=budget, stats=st)
        return st, (tmp_path / name).read_text()
    return go, passes


def _duck(monkeypatch, seqs):
    ref, asked = DuckReference(seqs), []

    def reference_for(ctx, path, contigs=None):
        asked.append((path, contigs))
        return ref
    monkeypatch.setattr(tasks, "reference_for", reference_for)
    return ref, asked


SEQS = {"ctg1": "ACGTRYACGT" * 35_000, "ctg2": "TTGCA" * 52_000}


@pytest.mark.parametrize("extra,contigs", [([], ["ctg1", "ctg2"]), (["--contig", "ctg2"], ["ctg2"]), (["--regions", "one.bed"], ["ctg1"])])
def test_reference_contigs_follow_the_plan(run, monkeypatch, caplog, extra, contigs):
    go, _ = run
    open("one.bed", "w").write("ctg1\t120000\t180000\n")
    ref, asked = _duck(monkeypatch, SEQS)
    caplog.set_level(logging.INFO)
    go((S4, extra + ["--reference", "genome.fa"]))
    assert asked == [("genome.fa", contigs)]
    assert "Opening for reading: genome.fa" in caplog.text


def test_no_reference_no_load(run, monkeypatch):
    go, passes = run
    ref, asked = _duck(monkeypatch, SEQS)
    st, text = go((S4, []))
    assert asked == [] and ref.prefetched == [] and st["prefetch_s"] == []
    assert "\tN\t<DEL>\t" in text


@pytest.mark.parametrize("extra", [[], ["--combine-max-inmemory-results", "1"]])
def test_writer_of_either_ordering_gets_the_reference(run, monkeypatch, extra):
    go, passes = run
    ref, _ = _duck(monkeypatch, SEQS)
    made = []
    orig = vcf.VCFWriter.__init__

    def init(self, config, handle, reference=None):
        made.append(reference)
        orig(self, config, handle, reference)
    monkeypatch.setattr(vcf.VCFWriter, "__init__", init)
    st, text = go((S4, extra + ["--reference", "genome.fa"]))
    assert made == [ref]
    records = [line.split("\t") for line in text.splitlines() if not line.startswith("#")]
    assert len(records) == 6
    for r in records:
        seq, pos, svtype = SEQS[r[0]], int(r[1]), r[7].split("SVTYPE=")[1].split(";")[0]
        ref = {"DEL": seq[pos - 1:pos + 150]}.get(svtype, seq[pos - 1].translate(vcf.AMBIGUOUS))
        alt = {"DEL": seq[pos - 1], "INS": ref + "ACGT" * 15, "DUP": "<DUP>".translate(vcf.AMBIGUOUS)}[svtype]
        assert r[3:5] == [ref, alt], r


@pytest.mark.parametrize("budget", [1, None])
def test_one_prefetch_per_pass_with_that_pass_calls(run, monkeypatch, budget):
    go, passes = run
    ref, _ = _duck(monkeypatch, SEQS)
    st, _ = go((S4, ["--reference", "genome.fa"]), budget=budget)
    assert st["passes"] == len(passes) == len(ref.prefetched) == len(st["prefetch_s"]) == len(st["prefetch_bytes"])
    assert st["passes"] == (2 if budget == 1 else 1)
    for (made, want), got in zip(passes, ref.prefetched):
        assert got == want and len(got) == 4 * len(made) // 3          # a DEL asks for two intervals, the INS and DUP for one each
    assert st["prefetch_bytes"] == [sum(e - s for _, s, e in p) for p in ref.prefetched]


def _fasta(path, kind):
    text = b"".join(b">%s\n%s\n" % (n.encode(), s[:1000].encode()) for n, s in SEQS.items())
    if kind == "gzip":
        text = gzip.compress(text)
    if kind != "missing":
        with open(path, "wb") as f:
            f.write(text)
    return path


@pytest.mark.parametrize("kind", ["gzip", "missing"])
def test_unreadable_fasta_leaves_the_output_as_without_it(run, caplog, tmp_path, kind):
    go, _ = run
    _, plain = go((S4, []), name="plain.vcf")
    path = _fasta(str(tmp_path / f"{kind}.fa.gz"), kind)
    caplog.clear()
    st, text = go((S4, ["--reference", path]), name="ref.vcf")
    errors = [r for r in caplog.records if r.levelno >= logging.ERROR]
    assert len(errors) == 1 and f"Unable to open reference file {path}" in errors[0].getMessage()
    assert text == plain and st["prefetch_s"] == []
