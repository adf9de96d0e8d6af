"""`python -m sniffles_b200.index IN.bam [-c | --csi] [-m | --min-shift N] [-o OUT] [--allow-overwrite]`: the BAI (default) or CSI
index of a coordinate-sorted BAM, built on the GPU (bamio.build_index), with the options of `samtools index`.  Writes IN.bam.bai /
IN.bam.csi, or OUT; an existing output is refused unless --allow-overwrite is given.  An input that is not a BGZF BAM, is truncated,
fails a block's CRC-32 or is not sorted by coordinate exits with status 1 and one fatal-error line naming the block or the record;
nothing is written then."""
import argparse
import logging
import os
import struct
import sys

log = logging.getLogger("sniffles_b200.index")


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m sniffles_b200.index", description="Index a coordinate-sorted BAM on the GPU (.bai, or .csi with -c).")
    ap.add_argument("input", help="the coordinate-sorted BAM file")
    ap.add_argument("-c", "--csi", action="store_true", help="write a CSI index (default: BAI)")
    ap.add_argument("-m", "--min-shift", type=int, default=None, help="CSI: the width of the smallest bins, 2^N (default 14); implies -c")
    ap.add_argument("-o", "--output", default=None, help="the index file (default: INPUT.bai or INPUT.csi)")
    ap.add_argument("--allow-overwrite", action="store_true", help="replace an existing index file")
    ap.add_argument("--device", type=int, default=0, help="the CUDA device")
    a = ap.parse_args(argv)
    csi = a.csi or a.min_shift is not None
    min_shift = 14 if a.min_shift is None else a.min_shift
    out = a.output or a.input + (".csi" if csi else ".bai")

    def fatal(msg):
        log.error(f"{msg} (Fatal error, exiting.)")
        return 1
    if not 1 <= min_shift <= 31:
        return fatal(f"--min-shift {min_shift}: must be in 1..31")
    if not os.path.exists(a.input):
        return fatal(f"Input file '{a.input}' does not exist.")
    if os.path.exists(out) and not a.allow_overwrite:
        return fatal(f"Output file '{out}' already exists! Use --allow-overwrite to ignore this check and overwrite.")
    from . import bamio, binding
    try:
        data = bamio.build_index(a.input, "csi" if csi else "bai", min_shift, device=a.device)
    except (ValueError, struct.error, binding.SnfbError) as e:
        return fatal(f"Unable to index '{a.input}': {e}")
    tmp = out + ".tmp"
    with open(tmp, "wb") as f:
        f.write(data)
    os.replace(tmp, out)
    log.info(f"Wrote {out} ({len(data)} bytes)")
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(name)s (%(process)d): %(message)s", stream=sys.stdout)
    sys.exit(main())
