"""Population annotation on the device: the command line against the reference's combine runs with --combine-population
(tests/golden/population), snfb_population_match against the reference's picks and against the oracle on a seeded fuzz."""
import gzip
import os
import random

import pytest

import combine_cli_common as ccc
import population_common as pc
from oracle import population as opop
from sniffles_b200 import __main__ as cli, combine_run, tasks
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

POPS, GOLD = pc.load_expected()


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    return ccc.write_inputs(str(tmp_path_factory.mktemp("population_inputs")))


@pytest.fixture(scope="module")
def ctx():
    return tasks.device_context(0)


def _lines(path):
    data = open(path, "rb").read()
    return ccc.vcf_lines((gzip.decompress(data) if path.endswith(".gz") else data).decode())


@pytest.mark.parametrize("label", sorted(GOLD))
def test_command_line_matches_the_reference(label, inputs, tmp_path, monkeypatch):
    case = GOLD[label]
    monkeypatch.chdir(inputs)
    out = str(tmp_path / "out.vcf")
    assert cli.main(pc.case_args(case, inputs, out)) == 0
    assert _lines(out) == case["vcf"]


@pytest.mark.parametrize("label", ["default4", "strict_alignment4", "regions", "tmpfile"])
def test_pass_budgets_and_bgzip(label, inputs, tmp_path, monkeypatch):
    case = GOLD[label]
    monkeypatch.chdir(inputs)
    for budget in (1, 10 ** 9):
        out = str(tmp_path / f"b{budget}.vcf")
        st = {}
        combine_run.combine_snfs(sconfig.SnifflesConfig(*pc.case_args(case, inputs, out)), budget=budget, stats=st)
        assert _lines(out) == case["vcf"]
        assert st["population_s"] > 0 and st["population_match_s"] > 0
        if budget == 1:
            assert st["passes"] >= 2
    if label != "tmpfile":                         # above --combine-max-inmemory-results a .vcf.gz is written plain
        gz = str(tmp_path / "out.vcf.gz")
        assert cli.main(pc.case_args(case, inputs, gz)) == 0
        assert _lines(gz) == case["vcf"] and os.path.getsize(gz + ".tbi") > 0


def _load(ctx, t):
    ctx.population_load(t["contig"], t["block"], t["svtype"], t["pos"], t["svlen"], t["alt"])


def _match(ctx, q, s):
    return ctx.population_match(q["contig"], q["svtype"], q["pos"], q["svlen"], q["alt"], s["combine_match"], s["combine_match_max"], s["combine_pctseq"], 100_000)


def test_match_vectors_of_the_reference(ctx):
    table, q, sets = pc.load_vectors()
    _load(ctx, table)
    for s in sets:
        assert _match(ctx, q, s).tolist() == s["best"], s["combine_pctseq"]
    assert "population_match" in [n for n, _, _ in ctx.timings()]


def _fuzz(seed, n_var=50_000, n_q=100_000):
    """a seeded table and calls: 2 contigs of 40 blocks and variants of a contig absent from the run (-1); positions on a 10-bp grid
    (ties), at pos 0 and block edges, 3 % stored under a block their pos is not in; BND with svlen 0, DEL with negative svlen; INS ALTs
    longer than 2,048 bytes, with bytes outside ACGTN, <INS> and empty.  Calls: 85 % near a variant, the rest anywhere, some on a contig
    the table lacks (2) or no contig (-1)."""
    rng, bs = random.Random(seed), 100_000
    seq = lambda n: bytes(rng.choice(b"ACGT") for _ in range(n))

    def alt_for(st, svlen):
        r = rng.random()
        if st != 0:
            return b"<" + pc.TYPES[st].encode() + b">" if r < 0.9 else b""
        return b"<INS>" if r < 0.05 else b"" if r < 0.08 else seq(2049 + rng.randrange(1200)) if r < 0.1 else seq(max(1, svlen))
    t = {k: [] for k in ("contig", "block", "svtype", "pos", "svlen", "alt")}
    for _ in range(n_var):
        b, st, r = rng.randrange(40), rng.choice([0, 0, 1, 1, 2, 3, 4]), rng.random()
        pos = b * bs + (rng.randrange(40) if r < 0.1 else bs - 1 - rng.randrange(40) if r < 0.2 else rng.randrange(bs // 10) * 10)
        pos += rng.choice([-bs, bs]) // 2 if rng.random() < 0.03 else 0
        svlen = 0 if st == 4 else rng.choice([20, 30, 50, 100, 300, 1000]) * (-1 if st == 1 else 1)
        alt = bytearray(alt_for(st, svlen))
        if alt[:1] not in (b"", b"<") and rng.random() < 0.1:
            alt[rng.randrange(len(alt))] = rng.choice(b"acgtRYK*\x00\xff")
        for k, v in zip(t, (rng.choice([0, 0, 1, 1, -1]), b * bs, st, pos, svlen, bytes(alt))):
            t[k].append(v)
    q = {k: [] for k in ("contig", "svtype", "pos", "svlen", "alt")}
    for _ in range(n_q):
        if rng.random() < 0.85:
            i = rng.randrange(n_var)
            c, st, a = t["contig"][i], t["svtype"][i], bytearray(t["alt"][i])
            pos = max(0, t["pos"][i] + rng.choice([0, 0, 10, -10, rng.randrange(-400, 400)]))
            svlen = 0 if st == 4 else t["svlen"][i] + rng.choice([0, 0, 10, -10, rng.randrange(-100, 100)])
            for _ in range(rng.randrange(1 + len(a) // 3) if st == 0 and a[:1] not in (b"", b"<") else 0):
                a[rng.randrange(len(a))] = rng.choice(b"ACGTN")
            alt = bytes(a)
        else:
            c, st = rng.choice([0, 1, 2, -1]), rng.randrange(5)
            pos = rng.choice([0, rng.randrange(40) * bs, rng.randrange(40 * bs)])
            svlen = 0 if st == 4 else rng.choice([0, 20, 50, 100]) * (-1 if st == 1 else 1)
            alt = alt_for(st, svlen)
        svlen = 1 if st == 0 and svlen == 0 else svlen          # zero-length INS calls have their own test
        for k, v in zip(q, (c, st, pos, svlen, alt)):
            q[k].append(v)
    return t, q


def test_fuzz_against_the_oracle(ctx):
    t, q = _fuzz(11)
    _load(ctx, t)
    n = len(q["pos"])
    sets = [dict(combine_match=250, combine_match_max=1000, combine_pctseq=0.7), dict(combine_match=250, combine_match_max=1000, combine_pctseq=0.0),
            dict(combine_match=250, combine_match_max=1000, combine_pctseq=1.0), dict(combine_match=500, combine_match_max=30, combine_pctseq=0.7)]
    thirds = [(0, n // 3), (n // 3, 2 * n // 3), (2 * n // 3, n - 5000), (n - 5000, n)]
    matched = 0
    for s, (a, b) in zip(sets, thirds):
        sub = {k: v[a:b] for k, v in q.items()}
        got = _match(ctx, sub, s).tolist()
        want = opop.match(t, sub, s["combine_match"], s["combine_match_max"], s["combine_pctseq"], 100_000)
        assert got == want, (s, next(i for i in range(len(got)) if got[i] != want[i]))
        matched += sum(x >= 0 for x in got)
    assert matched > n // 4


def test_zero_length_ins_is_reported(ctx):
    t = {"contig": [0, 0], "block": [0, 0], "svtype": [0, 0], "pos": [500, 500], "svlen": [30, 0], "alt": [b"A" * 30, b""]}
    _load(ctx, t)
    q = {"contig": [0, 0, 0], "svtype": [0, 0, 0], "pos": [500, 500, 510], "svlen": [0, 30, 0], "alt": [b"", b"A" * 30, b""]}
    s = dict(combine_match=250, combine_match_max=1000, combine_pctseq=0.7)
    got = _match(ctx, q, s).tolist()
    assert got == [-2, 0, -1] == opop.match(t, q, 250, 1000, 0.7, 100_000)
    assert _match(ctx, q, dict(s, combine_pctseq=0.0)).tolist() == [1, 0, -1]


def test_second_load_replaces_the_first(ctx):
    a = {"contig": [0], "block": [0], "svtype": [1], "pos": [1000], "svlen": [-100], "alt": [b"<DEL>"]}
    b = {"contig": [0, 0], "block": [0, 0], "svtype": [2, 1], "pos": [5000, 1010], "svlen": [100, -100], "alt": [b"<DUP>", b"<DEL>"]}
    q = {"contig": [0, 0], "svtype": [1, 2], "pos": [1000, 5000], "svlen": [-100, 100], "alt": [b"<DEL>", b"<DUP>"]}
    s = dict(combine_match=250, combine_match_max=1000, combine_pctseq=0.7)
    _load(ctx, a)
    assert _match(ctx, q, s).tolist() == [0, -1]
    _load(ctx, b)
    assert _match(ctx, q, s).tolist() == [1, 0]
    _load(ctx, {k: [] for k in a})
    assert _match(ctx, q, s).tolist() == [-1, -1]


def test_contig_absent_from_the_run(ctx):
    # a variant of a contig the run does not have (-1) is keyed past the table's contigs; a call on a contig the table lacks finds nothing
    t = {"contig": [0, -1], "block": [0, 0], "svtype": [1, 1], "pos": [1000, 1000], "svlen": [-100, -100], "alt": [b"<DEL>", b"<DEL>"]}
    _load(ctx, t)
    q = {"contig": [0, 1, 2, -1], "svtype": [1] * 4, "pos": [1000] * 4, "svlen": [-100] * 4, "alt": [b"<DEL>"] * 4}
    s = dict(combine_match=250, combine_match_max=1000, combine_pctseq=0.7)
    assert _match(ctx, q, s).tolist() == [0, -1, -1, -1] == opop.match(t, q, 250, 1000, 0.7, 100_000)
