"""Indexing a BAM (bamio.build_index, `python -m sniffles_b200.index`) without a GPU: the host restatement of the index tables against the
two htslib-written CSI fixtures (hg008.bam rebuilt with its original byte layout by bam_index_host.hg008_bam), the command line's
refusals that need no device, and the missing-index message of the call path."""
import logging
import os
import shutil
import struct

import pytest

import bam_index_host as H
from sniffles_b200 import __main__ as cli
from sniffles_b200 import bamio
from sniffles_b200 import index as index_cli

BAMS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams")


@pytest.mark.parametrize("name", ["hg002", "hg008"])
def test_host_restatement_matches_htslib_csi(name, tmp_path):
    """bins as a map, every chunk list, every bin's loffset, the pseudo-bins' offsets and counts, n_no_coor"""
    path = H.fixture_bam(name, tmp_path)
    with open(os.path.join(BAMS, name + ".bam.csi"), "rb") as f:
        want = H.parse_index(f.read())
    body, tab = H.host_index(path, "csi")
    got = H.parse_index(body)
    assert (got["min_shift"], got["depth"]) == (want["min_shift"], want["depth"]) == (14, 5)
    assert got["refs"] == want["refs"]
    assert got["n_no_coor"] == want["n_no_coor"]
    assert tab["n_records"] == {"hg002": 1, "hg008": 16}[name]


def test_hg008_parent_merge(tmp_path):
    """a naive build of hg008 has 7 bins with records; htslib's finishing rules move one small bin into its parent"""
    contigs, recs = H.rows(H.fixture_bam("hg008", tmp_path))
    naive = {(t, H._reg2bin(max(b, 0), e, 14, 5)) for t, b, e, *_ in recs if t >= 0}
    assert len(naive) == 7
    with open(os.path.join(BAMS, "hg008.bam.csi"), "rb") as f:
        assert sum(len([b for b in r if b != 37450]) for r in H.parse_index(f.read())["refs"]) == 6


def test_bai_and_csi_of_the_same_tables_agree(tmp_path):
    """the BAI and CSI bodies of one BAM hold the same bins and chunks (CSI adds loffsets, BAI the linear index)"""
    path = H.fixture_bam("hg008", tmp_path)
    bai, csi = H.parse_index(H.host_index(path, "bai")[0]), H.parse_index(H.host_index(path, "csi")[0])
    assert [{b: c for b, (_, c) in r.items()} for r in bai["refs"]] == [{b: c for b, (_, c) in r.items()} for r in csi["refs"]]
    assert len(bai["lin"]) == 218 and csi["lin"] is None


def _run_cli(args, caplog):
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="sniffles_b200.index"):
        code = index_cli.main(args)
    return code, [r for r in caplog.records if r.levelno >= logging.ERROR]


def test_cli_refuses_an_existing_output(tmp_path, caplog):
    bam = str(tmp_path / "x.bam")
    shutil.copyfile(os.path.join(BAMS, "hg002.bam"), bam)
    with open(bam + ".bai", "wb") as f:
        f.write(b"old")
    code, errs = _run_cli([bam], caplog)
    assert code == 1 and len(errs) == 1
    assert "already exists! Use --allow-overwrite" in errs[0].getMessage() and errs[0].getMessage().endswith("(Fatal error, exiting.)")
    with open(bam + ".bai", "rb") as f:
        assert f.read() == b"old"
    code, errs = _run_cli([bam, "-c", "-o", bam + ".bai"], caplog)
    assert code == 1 and len(errs) == 1


@pytest.mark.parametrize("kind", ["text", "gzip_not_bam", "truncated_header"])
def test_cli_refuses_input_that_is_not_a_bam(kind, tmp_path, caplog):
    bam = str(tmp_path / "x.bam")
    if kind == "text":
        data = b"@HD\tVN:1.6\nread1\t0\tchr1\t1\t60\t4M\t*\t0\t0\tACGT\t*\n"
    elif kind == "gzip_not_bam":
        data = bamio._bgzf_block(b"##fileformat=VCFv4.2\n") + bamio._BGZF_EOF
    else:
        head = b"BAM\1" + struct.pack("<i", 1000) + b"@HD\tVN:1.6\n"
        data = bamio._bgzf_block(head) + bamio._BGZF_EOF
    with open(bam, "wb") as f:
        f.write(data)
    for args, out in (([bam], bam + ".bai"), ([bam, "-c"], bam + ".csi")):
        code, errs = _run_cli(args, caplog)
        assert code == 1 and len(errs) == 1, kind
        assert errs[0].getMessage().startswith(f"Unable to index '{bam}'")
        assert not os.path.exists(out) and not os.path.exists(out + ".tmp")


def test_call_sample_without_an_index(tmp_path, caplog):
    """the reference's fatal message, plus the command that builds the index; no output is written"""
    bam = str(tmp_path / "noidx.bam")
    shutil.copyfile(os.path.join(BAMS, "hg002.bam"), bam)
    vcf_path = str(tmp_path / "out.vcf")
    with caplog.at_level(logging.ERROR):
        code = cli.main(["--input", bam, "--vcf", vcf_path])
    assert code == 1
    msgs = [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR]
    assert len(msgs) == 1
    assert msgs[0].startswith(f"Unable to load index for input file '{bam}'. Please verify that your input file is sorted + indexed")
    assert f"python -m sniffles_b200.index {bam}" in msgs[0]
    assert not os.path.exists(vcf_path)


def test_genotype_vcf_without_an_index(tmp_path, caplog):
    bam = str(tmp_path / "noidx.bam")
    shutil.copyfile(os.path.join(BAMS, "hg002.bam"), bam)
    targets = os.path.join(os.path.dirname(BAMS), "genotype", "basic.vcf")
    with caplog.at_level(logging.ERROR):
        code = cli.main(["--input", bam, "--vcf", str(tmp_path / "out.vcf"), "--genotype-vcf", targets])
    assert code == 1
    assert any(r.getMessage().startswith(f"Unable to load index for input file '{bam}'") for r in caplog.records)
