"""snfb_genotype_targets on the device against the plain-Python restatement (oracle/genotype.py) at scale, its launch count, that it
leaves the run's results alone, and the --genotype-vcf mode end to end through the device BAM ingest."""
import os

import numpy as np
import pytest
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from oracle import genotype as ogt
from sniffles_b200 import abi, bamio, binding, genotype, synth
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

NAMES = abi.SVTYPE_NAMES


def _sv(svtype, pos, svlen, first, mate, names):
    """a target column row as oracle/genotype.py reads it (mate contig by name; -1 = a name the header lacks)"""
    return ogt.Sv(NAMES[svtype] if svtype >= 0 else "CNV", pos, svlen, first, names[mate] if mate >= 0 else "unknown")


@pytest.fixture(scope="module")
def run2():
    blk = synth.config_block(2, 0.01)
    cfg_ns = sconfig.default_config()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg_ns))
    ctx.load(blk)
    n0 = ctx.launch_count()
    res = ctx.run()
    res.launches = ctx.launch_count() - n0          # snfb_run's launch count before any genotype call on the context
    yield blk, cfg_ns, ctx, res
    ctx.close()


def test_device_matches_oracle_at_scale(run2):
    blk, cfg_ns, ctx, res = run2
    rng = np.random.default_rng(7)
    cols = synth.genotype_targets(res.cand, len(blk.task), blk.task["contig_len"], rng, 200_000)
    match, cs, cc, ce, flag = ctx.genotype_targets(*cols, cfg_ns.combine_match, cfg_ns.combine_match_max)
    task = cols[0]
    ranges = np.searchsorted(res.cand["task"], np.arange(len(blk.task) + 1))
    from test_gpu_full_size import numpy_filter
    n_match, ok, span = 0, numpy_filter(blk, cfg_ns)[0], ogt.record_spans(blk)
    for t in np.unique(task):
        idx = np.nonzero(task == t)[0]
        lo, hi = int(ranges[t]), int(ranges[t + 1])
        cands = ogt.cand_svs(res.cand[lo:hi], blk.contig_names)
        targets = [_sv(*(int(cols[k][i]) for k in (1, 2, 3, 4, 5)), blk.contig_names) for i in idx]
        want = np.array([lo + m if m >= 0 else -1 for m in ogt.match(cands, targets, cfg_ns.combine_match, cfg_ns.combine_match_max, cfg_ns.cluster_merge_bnd)])
        assert np.array_equal(match[idx], want), int(t)
        n_match += int((want >= 0).sum())
        try:
            cov = ogt.coverage(targets, ogt.coverage_vector(blk, ok, span, int(t)), cfg_ns.coverage_binsize)
        except UnboundLocalError:
            assert flag[idx].any(), int(t)
            continue
        assert not flag[idx].any(), int(t)
        assert np.array_equal(np.stack([cs[idx], cc[idx], ce[idx]], 1), np.array(cov)), int(t)
    assert n_match > 10_000


def test_launch_count_and_run_unchanged(run2):
    blk, cfg_ns, ctx, res = run2
    cols = synth.genotype_targets(res.cand, len(blk.task), blk.task["contig_len"], np.random.default_rng(3), 5000)
    n0 = ctx.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        ctx.genotype_targets(*cols, cfg_ns.combine_match, cfg_ns.combine_match_max)
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    assert kernels and len(kernels) == ctx.launch_count() - n0
    n1 = ctx.launch_count()
    again = ctx.run()
    assert ctx.launch_count() - n1 == res.launches
    assert again.cand.tobytes() == res.cand.tobytes() and again.alt.tobytes() == res.alt.tobytes()      # bytes: stdev_len is NaN for a BND
    ctx.genotype_targets(*cols, cfg_ns.combine_match, cfg_ns.combine_match_max)
    n2 = ctx.launch_count()
    third = ctx.run()
    assert ctx.launch_count() - n2 == res.launches
    assert third.cand.tobytes() == res.cand.tobytes() and third.alt.tobytes() == res.alt.tobytes()


def test_genotype_vcf_end_to_end(tmp_path):
    """a BAM through the device ingest, targets made from the run's own candidates: every target written, the .vcf.gz input gives the
    same bytes, a task whose first target is a BND is left out"""
    blk = synth.config_block(1, 0.5)
    bam, _ = bamio.write_bam(str(tmp_path / "s.bam"), blk)
    cfg = sconfig.default_config()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    ctx.load(blk)
    res = ctx.run()
    ctx.close()
    name = blk.contig_names[0]
    lines = ["##fileformat=VCFv4.2", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS"]
    for i, c in enumerate(res.cand):
        sv = NAMES[int(c["svtype"])]
        if sv.startswith("SINGLE") or sv == "BND":
            continue
        lines.append(f"{name}\t{int(c['pos']) + 1 + i % 7}\tt{i}\tN\t<{sv}>\t.\tPASS\tSVTYPE={sv};SVLEN={int(c['svlen'])}\tGT\t0/1")
    src = tmp_path / "t.vcf"
    src.write_text("\n".join(lines) + "\n")
    gz = str(tmp_path / "t.vcf.gz")
    data = src.read_bytes()
    with open(gz, "wb") as f:
        f.write(bamio._bgzf_block(data, 6) + bamio._BGZF_EOF)
    outs = []
    for inp in (str(src), gz):
        out = tmp_path / f"out{len(outs)}.vcf"
        c = sconfig.default_config("--input", bam, "--genotype-vcf", inp, "--vcf", str(out), "--all-contigs")
        c.input = bam
        n = genotype.genotype_vcf(c)
        assert n == len(lines) - 2
        outs.append(out.read_text())
    assert outs[0] == outs[1]
    recs = [l.split("\t") for l in outs[0].splitlines() if not l.startswith("#")]
    assert sum(r[9].split(":")[0] not in ("./.", "0/0") for r in recs) > 0.8 * len(recs)
    # a BND before any other target of the task: the task fails and nothing is written for it
    bad = tmp_path / "bnd_first.vcf"
    bad.write_text("\n".join(lines[:2] + [f"{name}\t5000\tb\tN\tN[{name}:9000[\t.\tPASS\tSVTYPE=BND\tGT\t0/1"] + lines[2:]) + "\n")
    c = sconfig.default_config("--input", bam, "--genotype-vcf", str(bad), "--vcf", str(tmp_path / "o.vcf"), "--all-contigs")
    c.input = bam
    assert genotype.genotype_vcf(c) == 0


@pytest.mark.parametrize("name", ["c1_ont_1mb", "phased_phase", "c3_hifi_mosaic", "hg008"])
def test_genotype_vcf_matches_reference(name, tmp_path):
    """the reference's GenotypeTask output (tests/golden/genotype), header included, from a BAM of the fixture block through the device
    ingest, the device run and snfb_genotype_targets"""
    import test_genotype_parity as tgp
    fx, blk = tgp.load(name)
    bam, _ = bamio.write_bam(str(tmp_path / "s.bam"), blk)
    extra = ["--input", bam, "--vcf", str(tmp_path / "out.vcf")]
    if len(blk.tr):              # the block's repeats are padded intervals: a BED that load_tandem_repeats pads back to them
        pad = sconfig.default_config().tandem_repeat_region_pad
        with open(tmp_path / "tr.bed", "w") as f:
            for t in range(len(blk.task)):
                o, n = int(blk.task[t]["tr_off"]), int(blk.task[t]["tr_n"])
                for k in range(n):
                    a, b = int(blk.tr[2 * (o + k)]), int(blk.tr[2 * (o + k) + 1])
                    f.write(f"{blk.contig_names[int(blk.task[t]['contig'])]}\t{a + pad if a > 0 else pad}\t{b - pad}\n")
        extra += ["--tandem-repeats", str(tmp_path / "tr.bed")]
    cfg = tgp.config_for(fx, *extra)
    cfg.input = bam
    assert genotype.genotype_vcf(cfg) == fx["n_written"]
    assert (tmp_path / "out.vcf").read_text() == fx["output"]
