"""`python -m sniffles_b200.sort IN.bam -o OUT.bam [--write-index] [--allow-overwrite] [--device N]`: the BAM sorted by coordinate on the
GPU (bamio.sort_bam), in `samtools sort`'s record order and BGZF member layout.  The output is written to OUT.bam.tmp and renamed when
complete; --write-index also writes OUT.bam.csi (min_shift 14, what `samtools sort --write-index` writes) with bamio.build_index.  An
existing output is refused unless --allow-overwrite is given, and so is an output naming the input.  An input that is not a BGZF BAM, is
truncated, fails a block's CRC-32 or holds a record that is not a valid BAM record exits with status 1 and one fatal-error line naming the
block or the record; nothing is left behind then.  Nothing is written to stdout."""
import argparse
import logging
import os
import struct
import sys

log = logging.getLogger("sniffles_b200.sort")


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m sniffles_b200.sort", description="Sort a BAM by coordinate on the GPU.")
    ap.add_argument("input", help="the BAM file")
    ap.add_argument("-o", "--output", required=True, help="the sorted BAM file")
    ap.add_argument("--write-index", action="store_true", help="also write OUTPUT.csi")
    ap.add_argument("--allow-overwrite", action="store_true", help="replace an existing output file")
    ap.add_argument("--device", type=int, default=0, help="the CUDA device")
    a = ap.parse_args(argv)
    out = a.output
    idx = out + ".csi"

    def fatal(msg):
        log.error(f"{msg} (Fatal error, exiting.)")
        return 1
    if not os.path.exists(a.input):
        return fatal(f"Input file '{a.input}' does not exist.")
    if os.path.abspath(a.input) == os.path.abspath(out) or (os.path.exists(out) and os.path.samefile(a.input, out)):
        return fatal(f"Output file '{out}' is the input file.")
    for p in (out, idx) if a.write_index else (out,):
        if os.path.exists(p) and not a.allow_overwrite:
            return fatal(f"Output file '{p}' already exists! Use --allow-overwrite to ignore this check and overwrite.")
    from . import bamio, binding
    tmp = out + ".tmp"
    try:
        bamio.sort_bam(a.input, tmp, device=a.device)
        index = bamio.build_index(tmp, "csi", 14, device=a.device) if a.write_index else None
    except (ValueError, struct.error, OSError, binding.SnfbError) as e:
        if os.path.exists(tmp):
            os.remove(tmp)
        return fatal(f"Unable to sort '{a.input}': {e}")
    os.replace(tmp, out)
    if index is not None:
        with open(idx + ".tmp", "wb") as f:
            f.write(index)
        os.replace(idx + ".tmp", idx)
    log.info(f"Wrote {out}" + (f" and {idx}" if index is not None else ""))
    return 0


if __name__ == "__main__":
    logging.basicConfig(level=logging.INFO, format="%(asctime)s %(levelname)s %(name)s (%(process)d): %(message)s", stream=sys.stderr)
    sys.exit(main())
