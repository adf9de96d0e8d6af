"""Sorting a BAM (bamio.sort_bam, `python -m sniffles_b200.sort`) without a GPU: the host restatement's member cuts against the htslib-written
hg008.bam's layout, its order against hg008's own record order, the header rewrite, and the command line's refusals that need no device."""
import json
import logging
import os
import struct

import pytest

import bam_index_host as IH
import bam_sort_host as H
from sniffles_b200 import abi, bamio
from sniffles_b200 import sort as sort_cli

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_member_cuts_reproduce_hg008_layout():
    """htslib's writer rule, from the header length and the 16 block_sizes, gives the 58 data members of the htslib-written hg008.bam"""
    with open(os.path.join(GOLDEN, "bams", "hg008_layout.json")) as f:
        lay = json.load(f)
    isizes = [i for _, i in lay["members"]]
    assert isizes[-1] == 0                                              # the EOF marker
    got = H.member_sizes(isizes[0], [4 + b for b in lay["block_size"]])
    assert got == isizes[:-1] and len(got) == 58
    assert max(lay["block_size"]) > 0xff00                              # records span members


def test_restatement_of_shuffled_hg008_gives_back_hg008(tmp_path):
    """hg008's records shuffled (tied records keep their relative order) come back in hg008's order, with its member layout"""
    src = IH.hg008_bam(str(tmp_path / "hg008.bam"))
    shuf = H.shuffled_bam(src, str(tmp_path / "shuf.bam"), seed=3)
    header, recs = H.records(src)
    _, srecs = H.records(shuf)
    assert srecs != recs and sorted(srecs) == sorted(recs)
    data, sizes = H.sorted_stream(shuf)
    assert data == header + b"".join(recs)
    assert sizes == [i for i, _ in H.members(src)][:-1]


def test_hg008_breaks_strand_ties_as_samtools(tmp_path):
    """the htslib-written file puts (17, 21493609) forward twice before reverse twice, and the same at contig 22"""
    _, recs = H.records(IH.hg008_bam(str(tmp_path / "hg008.bam")))
    keys = [struct.unpack_from("<ii", r, 4) + ((struct.unpack_from("<H", r, 18)[0] >> 4) & 1,) for r in recs]
    assert keys[keys.index((17, 21493609, 0)):][:4] == [(17, 21493609, 0)] * 2 + [(17, 21493609, 1)] * 2
    assert [k for k in keys if k[0] == 22] == sorted(k for k in keys if k[0] == 22)


def _header(text, refs=(("chr1", 1000),)):
    body = struct.pack("<i", len(refs)) + b"".join(struct.pack("<i", len(n) + 1) + n.encode() + b"\0" + struct.pack("<i", ln) for n, ln in refs)
    return b"BAM\1" + struct.pack("<i", len(text)) + text + body


@pytest.mark.parametrize("text,want", [
    (b"@HD\tVN:1.6\tSO:unsorted\n@SQ\tSN:chr1\tLN:1000\n", b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:1000\n"),
    (b"@HD\tVN:1.6\tSO:queryname\tGO:query\n@CO\tx\n", b"@HD\tVN:1.6\tSO:coordinate\tGO:query\n@CO\tx\n"),
    (b"@HD\tVN:1.4\n@SQ\tSN:chr1\tLN:1000\n", b"@HD\tVN:1.4\tSO:coordinate\n@SQ\tSN:chr1\tLN:1000\n"),
    (b"@SQ\tSN:chr1\tLN:1000\n@PG\tID:x\n", b"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:chr1\tLN:1000\n@PG\tID:x\n"),
    (b"", b"@HD\tVN:1.6\tSO:coordinate\n"),
])
def test_header_rewrite(text, want):
    """SO:coordinate replaces the @HD line's SO or is appended to it; without @HD a new line goes first; the rest is kept byte for byte"""
    got = bamio.sort_header(_header(text))
    assert got == _header(want)
    assert H.rewrite_header(_header(text)) == got


def test_sort_structs_match_the_library_sizes():
    L = pytest.importorskip("sniffles_b200.binding").lib()
    import ctypes as C
    assert (L.snfb_sizeof(19), L.snfb_sizeof(20)) == (C.sizeof(abi.SortInput), C.sizeof(abi.SortView))


def _run_cli(args, caplog):
    caplog.clear()
    with caplog.at_level(logging.INFO, logger="sniffles_b200.sort"):
        code = sort_cli.main(args)
    return code, [r for r in caplog.records if r.levelno >= logging.ERROR]


def _assert_refused(code, errs, want):
    assert code == 1 and len(errs) == 1
    msg = errs[0].getMessage()
    assert want in msg and msg.endswith("(Fatal error, exiting.)"), msg


def test_cli_refuses_a_missing_input(tmp_path, caplog):
    out = str(tmp_path / "s.bam")
    _assert_refused(*_run_cli([str(tmp_path / "none.bam"), "-o", out], caplog), "does not exist")
    assert os.listdir(tmp_path) == []


def test_cli_refuses_an_existing_output(tmp_path, caplog):
    bam, out = IH.hg008_bam(str(tmp_path / "x.bam")), str(tmp_path / "s.bam")
    with open(out, "wb") as f:
        f.write(b"old")
    _assert_refused(*_run_cli([bam, "-o", out], caplog), "already exists! Use --allow-overwrite")
    with open(out, "rb") as f:
        assert f.read() == b"old"
    os.remove(out)
    with open(out + ".csi", "wb") as f:
        f.write(b"old")
    _assert_refused(*_run_cli([bam, "-o", out, "--write-index"], caplog), "already exists! Use --allow-overwrite")
    assert sorted(os.listdir(tmp_path)) == ["s.bam.csi", "x.bam"]


def test_cli_refuses_the_input_as_output(tmp_path, caplog):
    bam = IH.hg008_bam(str(tmp_path / "x.bam"))
    before = open(bam, "rb").read()
    for out in (bam, os.path.join(str(tmp_path), ".", "x.bam")):
        _assert_refused(*_run_cli([bam, "-o", out, "--allow-overwrite"], caplog), "is the input file")
    assert open(bam, "rb").read() == before and os.listdir(tmp_path) == ["x.bam"]


@pytest.mark.parametrize("kind", ["text", "truncated_header"])
def test_cli_refuses_input_that_is_not_a_bam(kind, tmp_path, caplog):
    bam, out = str(tmp_path / "x.bam"), str(tmp_path / "s.bam")
    data = b"@HD\tVN:1.6\n" if kind == "text" else bamio._bgzf_block(b"BAM\1" + struct.pack("<i", 1000) + b"@HD\tVN:1.6\n") + bamio._BGZF_EOF
    with open(bam, "wb") as f:
        f.write(data)
    _assert_refused(*_run_cli([bam, "-o", out, "--write-index"], caplog), f"Unable to sort '{bam}'")
    assert os.listdir(tmp_path) == ["x.bam"]
