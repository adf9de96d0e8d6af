"""A BGZF member that breaks one of the SAM spec's header rules (§4.1) is refused before anything is inflated, with the message of the
rule it breaks: by snfb_inflate_bgzf, which names the rule, and by the BAM index's window streamer, which names the member's file offset
and tells a member that is not BGZF from a file that ends inside one."""
import os
import re
import struct
import zlib

import numpy as np
import pytest

from sniffles_b200 import bamio, binding

pytestmark = pytest.mark.gpu

HG002 = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams", "hg002.bam")
DATA = b"ACGTTGCA" * 300


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    yield c
    c.close()


def _member(data=DATA, xtra=None, isize=None) -> bytes:
    """one gzip member of `data` whose extra field is `xtra` (default: the BC subfield with the member's BSIZE) and whose ISIZE is `isize`"""
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    payload = c.compress(data) + c.flush()
    if xtra is None:
        xtra = b"BC" + struct.pack("<HH", 2, 12 + 6 + len(payload) + 8 - 1)
    head = bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff]) + struct.pack("<H", len(xtra)) + xtra
    return head + payload + struct.pack("<II", zlib.crc32(data), len(data) if isize is None else isize)


NOT_BGZF = "not a BGZF block (gzip member with an extra field expected)"
GOOD = _member()
CASES = {
    "not_gzip": (b"\x1f\x8c" + GOOD[2:], NOT_BGZF),
    "no_fextra": (GOOD[:3] + b"\x00" + GOOD[4:], NOT_BGZF),
    "under_18_bytes": (GOOD[:17], NOT_BGZF),
    "xlen_past_the_end": (GOOD[:10] + struct.pack("<H", 400) + bytes(20), "truncated BGZF header"),
    "no_bc_subfield": (_member(xtra=b"XY" + struct.pack("<H", 2) + bytes(2)), "BGZF block without a BC field or truncated"),
    "bsize_below_the_header": (_member(xtra=b"BC" + struct.pack("<HH", 2, 10)), "BGZF block without a BC field or truncated"),
    "ends_inside_the_member": (GOOD[:-5], "BGZF block without a BC field or truncated"),
    "isize_over_64k": (_member(isize=65537), "BGZF block claims more than 64 KiB of data"),
}


def test_good_members_inflate(ctx):
    assert ctx.inflate_bgzf(np.frombuffer(GOOD * 3, "u1")) == DATA * 3


@pytest.mark.parametrize("case", sorted(CASES))
def test_broken_member_is_refused_by_its_rule(ctx, case):
    bad, msg = CASES[case]
    with pytest.raises(binding.SnfbError, match=re.escape(f"snfb_inflate_bgzf: {msg}") + "$"):
        ctx.inflate_bgzf(np.frombuffer(GOOD + bad, "u1"))


@pytest.mark.parametrize("case", ["not_gzip", "isize_over_64k"])
def test_index_names_the_member_that_is_not_bgzf(ctx, case, tmp_path):
    with open(HG002, "rb") as f:
        z = bytearray(f.read())
    o, _, _, _ = list(bamio.bgzf_members(bytes(z)))[1]         # the first member after the header's
    if case == "not_gzip":
        z[o + 1] ^= 0xff
    else:
        bsize = struct.unpack_from("<H", z, o + 16)[0] + 1
        struct.pack_into("<I", z, o + bsize - 4, 65537)
    path = str(tmp_path / "bad.bam")
    with open(path, "wb") as f:
        f.write(bytes(z))
    with pytest.raises(binding.SnfbError, match=re.escape(f"not a BGZF block at file offset {o}: not a BGZF-compressed BAM file")):
        bamio.build_index(path, "bai", ctx=ctx)
