"""--output-rnames on the device: call_sample's RNAMES and SNF rnames against the unmodified reference (tests/golden/rnames/, names compared
as sets: the reference's order depends on PYTHONHASHSEED), the same files at every pass budget and at two ranks, snfb_read_names against a
host restatement on blocks with chosen read names (host reader and device ingest alike), the launches of a run without the option, and
combine mode over SNFs that carry names."""
import json
import os

import numpy as np
import pytest

import call_sample_common as csc
import ranks_common
import rnames_common as rnc
from sniffles_b200 import abi, bamio, binding, call, combine_run, synth, tasks
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

with open(rnc.EXPECTED) as _f:
    GOLD = json.load(_f)


def _config(case, paths, out_dir, *extra):
    args = rnc.case_args(case, paths, os.path.join(out_dir, "out.vcf"), os.path.join(out_dir, "out.snf"))
    cfg = sconfig.SnifflesConfig(*args, *extra)
    for k, v in GOLD["stamp"].items():
        setattr(cfg, k, v)
    return cfg


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    d = tmp_path_factory.mktemp("rnames_inputs")
    return {name: csc.write_inputs(name, str(d / name)) for name in {n for n, _ in rnc.CASES.values()}}


def _outputs(d):
    snf_path = os.path.join(d, "out.snf")
    return (open(os.path.join(d, "out.vcf"), "rb").read(), rnc.snf_form(snf_path) if os.path.exists(snf_path) else None)


@pytest.mark.parametrize("case", sorted(rnc.CASES))
def test_call_sample_names_equal_the_reference(case, inputs, tmp_path):
    gold = GOLD["cases"][case]
    cfg = _config(case, inputs[gold["input"]], str(tmp_path))
    stats = {}
    assert call.call_sample(cfg, stats=stats) == gold["n_written"]
    vcf_text, snf_form = _outputs(str(tmp_path))
    got = rnc.vcf_form(vcf_text.decode())
    assert got == gold["vcf"]
    assert all(r[4] is not None for r in got["records"])                  # an RNAMES entry on every record
    if "snf" in gold:
        assert snf_form == gold["snf"]
    assert len(stats["rnames_s"]) == stats["passes"]


@pytest.mark.parametrize("case", ["rn_c3_mosaic", "rn_phased_all_contigs", "rn_hg002_all_contigs"])
def test_every_budget_and_two_ranks_give_the_same_files(case, inputs, tmp_path):
    gold = GOLD["cases"][case]
    paths = inputs[gold["input"]]
    one = tmp_path / "one"
    one.mkdir()
    call.call_sample(_config(case, paths, str(one)), budget=1 << 40)
    bam = bamio.BamFile(paths["bam"])
    total = sum(it.inflated for it in call.task_inputs(bam, tasks.plan(bam.contigs, _config(case, paths, str(one)))[1]))
    bam.close()
    quarter = tmp_path / "quarter"
    quarter.mkdir()
    stats = {}
    call.call_sample(_config(case, paths, str(quarter)), budget=max(1, total // 4), stats=stats)
    assert stats["passes"] >= 2
    ranks = tmp_path / "ranks"
    ranks.mkdir()
    got = ranks_common.run_ranks(_rank_run, 2, case, paths, str(ranks))
    assert all(ok for ok, _ in got), got
    assert _outputs(str(one)) == _outputs(str(quarter)) == _outputs(str(ranks))


def _rank_run(rank, world, case, paths, out_dir):
    return call.call_sample(_config(case, paths, out_dir, "--gpus", str(world)), device=0, budget=1 << 22)


def test_a_run_without_the_option_launches_what_it_did(inputs, tmp_path):
    """the names step launches only when asked: a pass with it adds k_resolve, the three scan kernels and k_copy, nothing else changes"""
    case = "rn_c1_snf"
    paths = inputs[GOLD["cases"][case]["input"]]
    ctx = tasks.device_context(0)
    counts, stats = [], []
    for k, extra in enumerate(([], [], ["--output-rnames"])):
        d = tmp_path / str(k)
        d.mkdir()
        cfg = _config(case, paths, str(d))
        cfg.output_rnames = bool(extra)
        st = {}
        n0 = ctx.launch_count()
        call.call_sample(cfg, stats=st)
        counts.append(ctx.launch_count() - n0)
        stats.append(st)
    assert stats[1]["rnames_s"] == [] and len(stats[2]["rnames_s"]) == stats[2]["passes"] == 1
    assert counts[2] - counts[1] == 5
    assert b"RNAMES=" not in open(tmp_path / "1" / "out.vcf", "rb").read() and b"RNAMES=" in open(tmp_path / "2" / "out.vcf", "rb").read()


# ---- snfb_read_names on blocks with chosen read names
LONG_NAME = b"".join(bytes([33 + (k * 7) % 94]) for k in range(254)).replace(b"@", b"a")


def _qnames(rec, var):
    return [bytes(var[int(r["var_off"]):int(r["var_off"]) + int(r["l_qname"])]) for r in rec]


def _renamed(blk, args):
    """the block with the first supporting reads of its first two candidates renamed 'A' and LONG_NAME (every alignment of a read keeps
    one name); the var arena rebuilt around the new names, the SA text of every record kept"""
    names = _qnames(blk.rec, blk.var)
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(sconfig.default_config(*args)))
        ctx.load(blk)
        res = ctx.run()
    finally:
        ctx.close()
    picks = list(dict.fromkeys(names[int(res.cand_leads[int(c["lead_off"])]["rec"])] for c in res.cand))
    new = {picks[0]: b"A", picks[1]: LONG_NAME}
    parts, off = [], 0
    rec = blk.rec.copy()
    for i, r in enumerate(blk.rec):
        nm = new.get(names[i], names[i])
        sa = bytes(blk.var[int(r["var_off"]) + int(r["l_qname"]):int(r["var_off"]) + int(r["l_qname"]) + int(r["sa_len"])])
        rec[i]["var_off"], rec[i]["l_qname"] = off, len(nm)
        parts.append(nm + sa)
        off += len(nm) + len(sa)
    blk.rec, blk.var = rec, np.frombuffer(b"".join(parts) + b"\0" * 16, "u1").copy()
    blk.rec16 = blk.cigar16 = None
    return blk


def _want(res, rec, var):
    """per candidate: its hash list resolved on the host through the first of its leads carrying each hash"""
    out = []
    for i, c in enumerate(res.cand):
        lo, n = int(c["lead_off"]), int(c["lead_n"]) + int(c["long_n"])
        by_hash = {}
        for l in res.cand_leads[lo:lo + n]:
            by_hash.setdefault(int(l["qname_hash"]), _qnames(rec[int(l["rec"]):int(l["rec"]) + 1], var)[0].decode())
        out.append([by_hash[int(h)] for h in res.rnames[int(res.rn_off[i]):int(res.rn_off[i + 1])]])
    return out


def _check_block(blk, args, tmp_path):
    """host reader and device ingest: the names equal the restatement and each other; returns (result, names per candidate)"""
    cfg = abi.Config.from_sniffles(sconfig.default_config(*args))
    path = str(tmp_path / "named.bam")
    bamio.write_bam(path, blk)
    f = bamio.BamFile(path)
    regions = [(blk.contig_names[int(t["contig"])], int(t["start"]), int(t["end"])) for t in blk.task]
    bgzf, spans = f.device_input(regions)
    f.close()
    ctx = binding.Context(0)
    try:
        ctx.set_config(cfg)
        ctx.load(blk)
        host = ctx.run()
        hn = ctx.read_names()
        host_names = hn.per_candidate(host.rn_off, 0, len(host.cand))
        assert host_names == _want(host, blk.rec, blk.var) and hn.collisions == 0
        assert {"rnames_resolve", "rnames_copy"} <= {n for n, _, _ in ctx.timings()}
        ctx.load_bam(bgzf, spans, blk)
        dev = ctx.run()
        dn = ctx.read_names()
        rec, _, var, _ = ctx.ingest_fetch()
        dev_names = dn.per_candidate(dev.rn_off, 0, len(dev.cand))
        assert dev_names == _want(dev, rec, var)
    finally:
        ctx.close()
    key = ["task", "svtype", "pos", "end", "svlen", "support"]
    assert np.array_equal(host.cand[key], dev.cand[key]) and host_names == dev_names
    assert len(hn.off) == len(host.rnames) + 1 and len(hn.text) == hn.off[-1]
    return host, host_names


def test_names_of_chosen_reads(tmp_path):
    import test_oracle_golden as tog
    fx, blk = tog.load_fixture("c3_hifi_mosaic")
    args = fx["args"] + ["--long-ins-length", "500"]               # a 609-bp insertion then unions its leads_long's names
    res, names = _check_block(_renamed(blk, args), args, tmp_path)
    flat = {n for c in names for n in c}
    assert "A" in flat and LONG_NAME.decode() in flat
    assert all(len(c) == len(set(c)) == int(x["support"]) for c, x in zip(names, res.cand))
    # some read supports a candidate through several alignments (records): it is listed once, as the no-duplicates test above shows
    leads = [res.cand_leads[int(c["lead_off"]):int(c["lead_off"]) + int(c["lead_n"])] for c in res.cand]
    assert any(len(set(ll["rec"].tolist())) > len(set(ll["qname_hash"].tolist())) for ll in leads)
    # a long insertion whose extra names come only from leads_long
    extra = 0
    for c, n in zip(res.cand, names):
        lo, k, kl = int(c["lead_off"]), int(c["lead_n"]), int(c["long_n"])
        main = {int(l["qname_hash"]) for l in res.cand_leads[lo:lo + k]}
        extra += int(c["svtype"]) == abi.INS and kl > 0 and len(n) > len(main)
    assert extra > 0


def test_names_of_a_deep_block(tmp_path):
    blk = synth.generate(77, [300_000], 45.0, len_mean=12000.0, len_sd=3000.0, sv_spacing=6000.0, tr_frac=0.1)
    _, names = _check_block(_renamed(blk, []), [], tmp_path)
    assert max(len(c) for c in names) > 32


def test_a_pass_without_candidates(tmp_path):
    blk = synth.generate(5, [200_000], 20.0, len_mean=12000.0, len_sd=3000.0, sv_spacing=6000.0, tr_frac=0.0)
    empty = bamio.pack_records([(n, int(c["length"])) for n, c in zip(blk.contig_names, blk.contig)], [], [(0, 0, 200_000, 0)])
    ctx = binding.Context(0)
    try:
        ctx.set_config(abi.Config.from_sniffles(sconfig.default_config()))
        ctx.load(empty)
        res = ctx.run()
        rn = ctx.read_names()
    finally:
        ctx.close()
    assert len(res.cand) == 0 and len(rn.text) == 0 and list(rn.off) == [0] and rn.per_candidate(res.rn_off, 0, 0) == []


# ---- combine mode
def _combine(snfs, vcf_path):
    cfg = sconfig.SnifflesConfig("-i", *snfs, "-v", vcf_path, "--output-rnames")
    combine_run.combine_snfs(cfg)
    lines = [l for l in open(vcf_path).read().splitlines() if not l.startswith("#")]
    return rnc.combine_form(lines)


def test_combine_of_the_reference_snfs_keeps_their_order(tmp_path):
    got = _combine([os.path.join(rnc.GOLDEN, c + ".snf") for c in rnc.COMBINE_CASES], str(tmp_path / "c.vcf"))
    want = GOLD["combine"]["records"]
    assert [[r[0], r[1], r[4]] for r in got] == [[r[0], r[1], r[4]] for r in want]


def test_call_then_combine_gives_the_reference_names(inputs, tmp_path):
    snfs = []
    for case in rnc.COMBINE_CASES:
        d = tmp_path / case
        d.mkdir()
        cfg = _config(case, inputs[GOLD["cases"][case]["input"]], str(d))
        cfg.snf = str(d / (case + ".snf"))
        call.call_sample(cfg)
        snfs.append(cfg.snf)
    got = _combine(snfs, str(tmp_path / "c.vcf"))
    want = GOLD["combine"]["records"]
    assert [[r[0], r[1], sorted(r[4])] for r in got] == [[r[0], r[1], sorted(r[4])] for r in want]
