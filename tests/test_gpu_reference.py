"""--reference on the device: snfb_load_reference's unwrapped bytes and 'N' runs against a numpy restatement, the geometry and CRC
failures, snfb_fetch_reference against slicing, and end to end the reference's own masked candidates and VCF lines
(tests/golden/reference/golden.json, made by tests/golden/make_reference_golden.py)."""
import copy
import io
import json
import logging
import os

import numpy as np
import pytest

from sniffles_b200 import abi, bamio, binding, fasta, genotype, tasks, vcf
from sniffles_b200 import config as sconfig
import ref_fasta

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference", "golden.json")


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    yield c
    c.close()


def write(tmp_path, name, seqs, width=60, crlf=False, bgzf=False, block=0xff00):
    text = ref_fasta.fasta_text(seqs, width=width, crlf=crlf)
    path = tmp_path / name
    if bgzf:
        path.write_bytes(b"".join(bamio._bgzf_block(text[k:k + block]) for k in range(0, len(text), block)) + bamio._BGZF_EOF)
        (tmp_path / (name + ".fai")).write_bytes(ref_fasta.fai_text(seqs, width=width, crlf=crlf))
    else:
        path.write_bytes(text)
    return str(path)


def shapes(width, seed):
    rng = np.random.default_rng(seed)
    return [("empty", b""), ("one", b"N"), ("exact", ref_fasta.contig_seq(rng, 3 * width)), ("allN", b"N" * 70_001),
            ("big", ref_fasta.contig_seq(rng, 200_003)), ("small", ref_fasta.contig_seq(rng, 1_000))]


@pytest.mark.parametrize("fmt", ["plain", "crlf", "bgzf"])
@pytest.mark.parametrize("width", [1, 60, 61, 80, 4096])
def test_unwrap_and_n_runs_match_numpy(ctx, tmp_path, fmt, width):
    seqs = shapes(width, width)
    path = write(tmp_path, "r.fa" + (".gz" if fmt == "bgzf" else ""), seqs, width=width, crlf=fmt == "crlf", bgzf=fmt == "bgzf", block=4093)
    ref = fasta.Reference(path, ctx)
    runs = ref.n_runs()
    for name, s in seqs:
        assert ref.fetch(name) == s.decode(), (name, fmt, width)
        assert np.array_equal(runs[name].reshape(-1, 2), ref_fasta.n_runs(s)), (name, fmt, width)


def test_subset_of_contigs_from_bgzf(ctx, tmp_path):
    seqs = shapes(60, 3)
    path = write(tmp_path, "r.fa.gz", seqs, bgzf=True, block=2000)
    ref = fasta.Reference(path, ctx, contigs=["allN", "small"])
    assert {n for n, _, _ in ctx.timings()} >= {"h2d_ref", "inflate", "ref_unwrap", "ref_nruns"}
    assert ref.fetch("small") == seqs[5][1].decode() and set(ref.n_runs()) == {"allN", "small"}
    with pytest.raises(KeyError):
        ref.fetch("big", 0, 10)


def test_stale_fai_is_refused_naming_the_contig(ctx, tmp_path):
    seqs = shapes(60, 4)
    path = write(tmp_path, "r.fa", seqs, width=60)
    fai = ref_fasta.fai_text(seqs, width=60).decode().splitlines()
    fai[4] = fai[4].replace("\t60\t61", "\t61\t62")          # "big" written at 60 columns, indexed as 61
    (tmp_path / "r.fa.fai").write_text("\n".join(fai) + "\n")
    with pytest.raises(fasta.ReferenceError, match="sequence 'big'.*stale"):
        fasta.Reference(path, ctx)


def test_crc_flip_fails_the_load_and_the_task_runs_unmasked(ctx, tmp_path, caplog):
    seqs = [("ctg1", ref_fasta.contig_seq(np.random.default_rng(1), 200_000))]
    path = write(tmp_path, "r.fa.gz", seqs, bgzf=True, block=0xff00)
    z = bytearray(open(path, "rb").read())
    members = list(bamio.bgzf_members(bytes(z)))
    o1, _, _, _ = members[2]
    o2 = members[3][0]
    z[o2 - 8] ^= 0x10                                             # a CRC bit of member 2
    open(path, "wb").write(bytes(z))
    with pytest.raises(binding.SnfbError, match=f"block 2.*CRC32 mismatch.*byte {o1}"):
        fasta.Reference(path, ctx)
    from sniffles_b200 import synth
    blk = synth.generate(93, [200_000], 20.0, len_mean=9000.0, len_sd=2500.0, sv_spacing=6000.0)
    bam, _ = bamio.write_bam(str(tmp_path / "x.bam"), blk)
    plain = tasks.CallTask(id=0, sv_id=0, contig="ctg1", start=0, end=199_999, config=sconfig.default_config(), bam=bam).execute()[0]
    cfg = sconfig.default_config()
    cfg.reference = path
    with caplog.at_level(logging.ERROR):
        got = tasks.CallTask(id=0, sv_id=0, contig="ctg1", start=0, end=199_999, config=cfg, bam=bam).execute()[0]
    assert any("Unable to open reference file" in r.message and "CRC32" in r.message for r in caplog.records)
    assert [(c.svtype, c.pos, c.filter, c.genotypes) for c in got] == [(c.svtype, c.pos, c.filter, c.genotypes) for c in plain]


def test_fetch_matches_slicing(ctx, tmp_path):
    seqs = shapes(61, 9)
    path = write(tmp_path, "r.fa", seqs, width=61)
    ref = fasta.Reference(path, ctx)
    d = {n: s.decode() for n, s in seqs}
    rng = np.random.default_rng(17)
    iv = []
    for _ in range(10_000):
        n, s = seqs[int(rng.integers(1, len(seqs)))]
        L = len(s)
        a = int(rng.choice([rng.integers(0, L + 1), L - 1, L, max(0, L - 61), 60, 61, 0]))
        iv.append((n, a, a + int(rng.integers(0, 400))))
    ref.prefetch(iv)
    assert all(ref.fetch(n, a, b) == d[n][a:b] for n, a, b in iv)
    fresh = fasta.Reference(path, ctx)                        # single-query misses
    assert all(fresh.fetch(n, a, b) == d[n][a:b] for n, a, b in iv[:300])


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.parametrize("name", sorted(ref_fasta.GOLDEN_FASTA))
def test_calltask_with_reference_matches_reference_golden(name, tmp_path):
    from test_oracle_golden import load_fixture
    gold = _golden()["blocks"][name]
    fx, blk = load_fixture(name)
    bam, _ = bamio.write_bam(str(tmp_path / "s.bam"), blk)
    text, _ = ref_fasta.golden_fasta(name)
    assert ref_fasta.sha256(text) == gold["fasta_sha256"]
    fa = tmp_path / "ref.fa"
    fa.write_bytes(text)
    for key, entry in gold["args"].items():
        for device_ingest in (True, False):
            for t, (want, want_vcf) in enumerate(zip(gold["tasks"], entry["vcf"])):
                tk = blk.task[t]
                o, n = int(tk["tr_off"]), int(tk["tr_n"])
                tr = [(int(blk.tr[2 * (o + k)]), int(blk.tr[2 * (o + k) + 1])) for k in range(n)]
                cfg = sconfig.default_config(*entry["argv"])
                cfg.reference = str(fa)
                task = tasks.CallTask(id=int(tk["task_id"]), sv_id=0, contig=blk.contig_names[int(tk["contig"])], start=int(tk["start"]), end=int(tk["end"]),
                                      config=cfg, bam=bam, tandem_repeats=tr, device_ingest=device_ingest)
                task.build_leadtab()
                cands = task.call_candidates(True, cfg)
                res = task.block_run.result
                got = [[abi.SVTYPE_NAMES[int(c["svtype"])], *(int(c[k]) for k in ("pos", "end", "svlen", "support", "qual")), bool(c["precise"]), int(c["fwd"]), int(c["rev"]),
                        [int(c[k]) for k in ("cov_upstream", "cov_start", "cov_center", "cov_end", "cov_downstream")]] for c in res.cand]
                assert got == want["cands"], (name, key, t, device_ingest)
                assert want["cov_mean"] == float(res.task_cov_mean[0]) and want["read_count"] == int(res.task_read_count[0]), (key, t)
                final = task.finalize_candidates(cands, False, cfg)
                ref = tasks.reference_for(tasks.device_context(0), str(fa))
                ref.prefetch(vcf.reference_intervals(final, cfg))
                buf = io.StringIO()
                w = vcf.VCFWriter(cfg, buf, reference=ref)
                for c in final:
                    w.write_call(copy.deepcopy(c))
                assert [ref_fasta.vcf_digest(line) for line in buf.getvalue().splitlines()] == want_vcf, (name, key, t, device_ingest)


def test_genotype_vcf_with_reference_equals_the_numpy_mask(tmp_path, monkeypatch):
    import test_genotype_parity as tgp
    fx, blk = tgp.load("phased_phase")
    bam, _ = bamio.write_bam(str(tmp_path / "s.bam"), blk)
    text, seqs = ref_fasta.golden_fasta("phased_phase")
    fa = tmp_path / "ref.fa"
    fa.write_bytes(text)
    outs = []
    for mode in ("device", "numpy"):
        out = tmp_path / f"{mode}.vcf"
        cfg = tgp.config_for(fx, "--input", bam, "--vcf", str(out))
        cfg.input = bam
        if mode == "device":
            cfg.reference = str(fa)
        else:
            lengths = {n: len(s) for n, s in seqs}

            def numpy_mask(block, config, ctx):
                per = {t: [tuple(map(int, r)) for r in ref_fasta.n_runs(dict(seqs)[block.contig_names[int(k["contig"])]])]
                       for t, k in enumerate(block.task) if lengths.get(block.contig_names[int(k["contig"])], -1) >= int(k["end"])}
                block.set_n_mask(per)
                return block
            monkeypatch.setattr(tasks, "mask_block", numpy_mask)
        genotype.genotype_vcf(cfg)
        outs.append(out.read_text())
    assert outs[0] == outs[1] and outs[0].count("\n") > 10
