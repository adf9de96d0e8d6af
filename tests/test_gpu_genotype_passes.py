"""genotype.genotype_vcf in the device passes of call.call_sample: every golden force-calling fixture gives the reference's bytes in one
pass, at one task per pass and at two or more passes; on a four-contig sample with targets from the run's own candidates, plain and
bgzipped output, --regions over two contigs and a task that fails in a middle pass give the bytes of one pass."""
import gzip

import pytest

import call_sample_common as csc
import test_genotype_parity as tgp
from sniffles_b200 import abi, bamio, binding, call, genotype, synth
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu


def _sizes(cfg):
    """the inflated BAM bytes of every task with targets, in task order"""
    bam = bamio.BamFile(cfg.input)
    _, targets = genotype.read_targets(cfg.genotype_vcf)
    planned = [p[:4] for p in genotype.plan(bam.contigs, targets, cfg) if p[4]]
    sizes = [it.inflated for it in call.task_inputs(bam, planned, regions_by_contig=cfg.regions_by_contig)]
    bam.close()
    return sizes


def _budgets(sizes):
    """one pass, one task per pass and, with two or more tasks, a budget just under their total"""
    out = [1 << 40, 1]
    if len(sizes) >= 2:
        out.append(max(sum(sizes) - 1, max(sizes)))
    return out


def _passes(sizes, budget):
    return len(list(call.group_passes(sizes, budget, size=lambda n: n)))


@pytest.mark.parametrize("name", tgp.BLOCKS)
def test_golden_fixture_at_any_budget(name, tmp_path):
    """the BAM and tandem repeats of test_gpu_genotype.py::test_genotype_vcf_matches_reference, at every budget of _budgets"""
    fx, _ = tgp.load(name)
    paths = csc.write_inputs(name, str(tmp_path / "in"))
    extra = ["--input", paths["bam"]] + (["--tandem-repeats", paths["tr"]] if "tr" in paths else [])
    cfg = tgp.config_for(fx, *extra)
    cfg.input = paths["bam"]
    sizes = _sizes(cfg)
    assert sizes
    for k, budget in enumerate(_budgets(sizes)):
        out = tmp_path / f"out{k}.vcf"
        cfg = tgp.config_for(fx, *extra, "--vcf", str(out))
        cfg.input = paths["bam"]
        stats = {}
        assert genotype.genotype_vcf(cfg, budget=budget, stats=stats) == fx["n_written"]
        assert stats["passes"] == _passes(sizes, budget)
        assert stats["passes"] == 1 if k == 0 else stats["passes"] >= min(2, len(sizes))
        assert len(stats["load_bam_s"]) == len(stats["run_s"]) == len(stats["genotype_s"]) == stats["passes"]
        assert sum(stats["pass_inflated_bytes"]) == sum(sizes)
        assert out.read_text() == fx["output"], budget


@pytest.fixture(scope="module")
def sample(tmp_path_factory):
    """four 300 kb contigs, a BAM of them and the candidates of one device run over the block"""
    d = tmp_path_factory.mktemp("genotype_passes")
    blk = synth.generate(11, [300_000] * 4, 12.0, len_mean=8000.0, len_sd=3000.0, sv_spacing=6000.0, phased_frac=0.3, tr_frac=0.0)
    bam, _ = bamio.write_bam(str(d / "s.bam"), blk)
    cfg = sconfig.default_config()
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    ctx.load(blk)
    res = ctx.run()
    ctx.close()
    lines = {name: [] for name in blk.contig_names}
    for i, c in enumerate(res.cand):
        sv = abi.SVTYPE_NAMES[int(c["svtype"])]
        if sv.startswith("SINGLE") or sv == "BND":
            continue
        name = blk.contig_names[int(blk.task[int(c["task"])]["contig"])]
        lines[name].append((int(c["pos"]) + 1 + i % 7, f"t{i}\tN\t<{sv}>\t.\tPASS\tSVTYPE={sv};SVLEN={int(c['svlen'])}\tGT\t0/1"))
    return {"dir": d, "bam": bam, "names": blk.contig_names, "lines": lines}


def _targets(sample, path, bnd_first=None):
    """a target VCF, sorted by contig then position; bnd_first: a contig whose first target is a BND (its task fails)"""
    out = ["##fileformat=VCFv4.2", "#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\tS"]
    for name in sample["names"]:
        if name == bnd_first:
            out.append(f"{name}\t100\tb\tN\tN[{name}:9000[\t.\tPASS\tSVTYPE=BND\tGT\t0/1")
        out += [f"{name}\t{pos}\t{rest}" for pos, rest in sorted(sample["lines"][name], key=lambda x: x[0])]
    path.write_text("\n".join(out) + "\n")
    return str(path)


def _run(sample, targets, out, budget, *extra):
    cfg = sconfig.default_config("--input", sample["bam"], "--genotype-vcf", targets, "--vcf", str(out), "--all-contigs", *extra)
    cfg.input = sample["bam"]
    stats = {}
    n = genotype.genotype_vcf(cfg, budget=budget, stats=stats)
    return n, stats


def _records(text):
    return [l for l in text.splitlines() if not l.startswith("#")]


def test_four_contigs_at_any_budget_plain_and_bgzipped(sample, tmp_path):
    targets = _targets(sample, tmp_path / "t.vcf")
    cfg = sconfig.default_config("--input", sample["bam"], "--genotype-vcf", targets, "--all-contigs")
    cfg.input = sample["bam"]
    sizes = _sizes(cfg)
    assert len(sizes) == 4
    outs = []
    for budget in _budgets(sizes):
        d = tmp_path / str(budget)
        d.mkdir()
        n, stats = _run(sample, targets, d / "out.vcf", budget)
        assert stats["passes"] == _passes(sizes, budget)
        n_gz, stats = _run(sample, targets, d / "out.vcf.gz", budget)
        assert stats["passes"] == _passes(sizes, budget)
        with gzip.open(d / "out.vcf.gz", "rb") as f:
            text = f.read()
        assert n_gz == n and text == (d / "out.vcf").read_bytes()
        assert (d / "out.vcf.gz.tbi").stat().st_size > 0
        outs.append((n, text, (d / "out.vcf.gz").read_bytes(), (d / "out.vcf.gz.tbi").read_bytes()))
    assert [_passes(sizes, b) for b in _budgets(sizes)][1:] == [4, 2]
    assert outs[0] == outs[1] == outs[2]
    recs = _records(outs[0][1].decode())
    assert outs[0][0] == len(recs) and len({r.split("\t")[0] for r in recs}) >= 3


def test_regions_over_two_contigs(sample, tmp_path):
    targets = _targets(sample, tmp_path / "t.vcf")
    bed = tmp_path / "r.bed"
    a, b = sample["names"][1], sample["names"][2]
    bed.write_text(f"{a}\t10000\t150000\n{a}\t200000\t290000\n{b}\t50000\t250000\n")
    outs = []
    for budget in (1 << 40, 1):
        out = tmp_path / f"out{budget}.vcf"
        n, stats = _run(sample, targets, out, budget, "--regions", str(bed))
        outs.append((n, out.read_text()))
    assert outs[0] == outs[1] and outs[0][0] > 0


def test_failed_task_in_a_middle_pass(sample, tmp_path, caplog):
    good = tmp_path / "good.vcf"
    _run(sample, _targets(sample, tmp_path / "t.vcf"), good, 1 << 40)
    bad_contig = sample["names"][2]
    bad = _targets(sample, tmp_path / "bad.vcf", bnd_first=bad_contig)
    want = [r for r in _records(good.read_text()) if r.split("\t")[0] != bad_contig]
    outs = []
    for budget in (1 << 40, 1):
        out = tmp_path / f"bad{budget}.vcf"
        n, stats = _run(sample, bad, out, budget)
        assert n == len(want) and _records(out.read_text()) == want
        outs.append(out.read_bytes())
    assert stats["passes"] == 4 and outs[0] == outs[1]
    assert f"GenotypeTask(id=2, contig={bad_contig}" in caplog.text
