"""The shape of k_cigar_walk's work on a synthetic block, counted on the CPU (no GPU needed).

    python scripts/walk_shape.py [--config 2] [--scale 0.05]

Packs synth.config_block(config, scale) to CIGAR16 and follows the kernel's schedule: a warp takes a tile of 32 consecutive records
(one record below WALK_WIDE_MIN records), cuts each passing record's 16-byte groups into chunks of up to 16 groups and walks the tile's
chunks in rounds of 32, one chunk per lane.  Prints groups per chunk, chunks and load batches (8 groups) per round, the share of useful
lanes in the load loop, flagged chunks (holding an E word) and the flagged groups a round decodes, one group per lane in passes of 32.

"Passing" applies the read filters that need no CIGAR (mapping quality, secondary / excluded flags, an empty CIGAR); the kernel also
drops reads shorter than the minimum alignment length and outside their task, which this count keeps.
"""
import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sniffles_b200 import abi, synth  # noqa: E402
from sniffles_b200 import config as sconfig  # noqa: E402

CH, TILE_WIDE = 16, 32
WALK_WIDE_MIN = 32 * 132 * 4 * 8       # extract.cuh: 32 x WALK_BLOCKS x warps per block


def shape(blk, cfg):
    blk.pack16()
    r, c = blk.rec16, blk.cigar16
    n_rec = len(r)
    tile = TILE_WIDE if n_rec >= WALK_WIDE_MIN else 1
    ok = (r["mapq"] >= cfg.mapq) & ((r["flag"] & 256) == 0) & (r["n_cigar"] > 0)
    if cfg.exclude_flags:
        ok &= (r["flag"] & cfg.exclude_flags) == 0
    G = ((r["n_cigar"].astype(np.int64) + 7) >> 3) * ok
    nch = (G + CH - 1) // CH
    # chunks in walk order: record, then chunk index inside the record
    rec_of = np.repeat(np.arange(n_rec), nch)
    first = np.cumsum(nch) - nch
    k = np.arange(len(rec_of)) - first[rec_of]
    ng = np.minimum(CH, G[rec_of] - k * CH)
    g0 = (r["cigar_off"].astype(np.int64) >> 3)[rec_of] + k * CH
    # per group: an E word (base word, bit 14), an extension word (bit 15); per chunk via prefix sums over the arena's groups
    grp = c[: len(c) // 8 * 8].reshape(-1, 8)
    e_grp = ((grp & 0xC000) == 0x4000).any(axis=1)
    x_grp = (grp & 0x8000).any(axis=1)
    cs_e = np.concatenate([[0], np.cumsum(e_grp)])
    cs_x = np.concatenate([[0], np.cumsum(x_grp)])
    e_per_chunk = cs_e[g0 + ng] - cs_e[g0]
    x_per_chunk = cs_x[g0 + ng] - cs_x[g0]
    flagged = e_per_chunk > 0
    # rounds: the tile's chunks in order, 32 per round
    t_of = rec_of // tile
    t_first = np.cumsum(np.bincount(t_of, minlength=n_rec // tile + 1))
    t_first = np.concatenate([[0], t_first[:-1]])
    pos = np.arange(len(rec_of)) - t_first[t_of]
    t_rounds = (np.bincount(t_of, minlength=len(t_first)) + 31) // 32
    round_of = (np.cumsum(t_rounds) - t_rounds)[t_of] + pos // 32
    n_rounds = int(t_rounds.sum())
    batches = np.zeros(n_rounds, np.int64)
    np.maximum.at(batches, round_of, (ng + 7) // 8)
    fl_chunks = np.bincount(round_of, weights=flagged, minlength=n_rounds)
    fl_groups = np.bincount(round_of, weights=ng * flagged, minlength=n_rounds)
    n_chunks = len(rec_of)
    return {
        "records": n_rec, "tile": tile, "passing records": int(ok.sum()), "chunks": n_chunks, "rounds": n_rounds,
        "groups per chunk": ng.mean(),
        "chunks per round": n_chunks / n_rounds,
        "load batches of 8 groups per round": batches.mean(),
        "useful lanes in the load loop": ng.sum() / (batches.sum() * 8 * 32),
        "flagged chunks": flagged.mean(),
        "E groups per flagged chunk": e_per_chunk[flagged].mean() if flagged.any() else 0.0,
        "flagged chunks per round": fl_chunks.mean(),
        "flagged groups per round": fl_groups.mean(),
        "decode passes of 32 groups per round": np.ceil(fl_groups / 32).mean(),
        "rounds with no flagged chunk": (fl_chunks == 0).mean(),
        "chunks holding an extension word": (x_per_chunk > 0).mean(),
    }


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--config", type=int, default=2)
    ap.add_argument("--scale", type=float, default=0.05)
    ap.add_argument("--threads", type=int, default=0)
    args = ap.parse_args()
    blk = synth.config_block(args.config, args.scale, threads=args.threads, with_seq=False)
    cfg = abi.Config.from_sniffles(sconfig.default_config(*(["--mosaic"] if args.config == 3 else [])))
    print(f"config {args.config}, scale {args.scale}")
    for name, v in shape(blk, cfg).items():
        print(f"  {name:40s} {v:.3f}" if isinstance(v, float) else f"  {name:40s} {v}")


if __name__ == "__main__":
    main()
