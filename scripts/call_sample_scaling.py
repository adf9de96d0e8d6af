"""Whole-sample calling on 1, 2, 4 and 8 GPUs (capped at the visible devices): call.call_sample at each world size, one rank per device,
as `torchrun --nproc-per-node N -m sniffles_b200 ... --gpus N` runs it.  Prints one JSON line: the card and its power limit; per input and
world size the wall time of rank 0's call_sample (after a warm-up run in the same processes), every rank's split (tasks, index weight,
inflated bytes, read / load / run / finalize / format seconds), the LPT load max / mean over the index weights, the gather and write
times, and a sha256 of the output files compared with the one-rank run's.

    python scripts/call_sample_scaling.py [--inputs c6,c2] [--c2-scale 0.01] [--sizes 1,2,4,8] [--out FILE]

The inputs are those of scripts/call_sample_bench.py (make_input).  The SNF hash leaves out what a run stamps on the file: each gzip
member's write time and the header's `gpus`, `vcf` and `snf`."""
import argparse
import datetime
import gzip
import hashlib
import json
import multiprocessing as mp
import os
import socket
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def files_sha256(vcf_path, snf_path):
    """sha256 over the decompressed VCF text, its .tbi and the SNF without its write times and run stamps"""
    h = hashlib.sha256()
    with open(vcf_path, "rb") as f:
        h.update(gzip.decompress(f.read()))
    with open(vcf_path + ".tbi", "rb") as f:
        h.update(f.read())
    with open(snf_path, "rb") as f:
        header = json.loads(f.readline())
        body = bytearray(f.read())
    for k in ("gpus", "vcf", "snf"):
        header["config"].pop(k, None)
    for blocks in header["index"].values():
        for parts in blocks.values():
            for off, _ in parts:
                body[off + 4:off + 8] = b"\0\0\0\0"
    h.update(json.dumps(header, sort_keys=True).encode())
    h.update(bytes(body))
    return h.hexdigest()


def _rank(rank, world, port, bam, tmp, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch
    import torch.distributed as tdist
    from sniffles_b200 import call
    from sniffles_b200 import config as sconfig
    torch.cuda.set_device(rank)
    tdist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(hours=2))
    try:
        out = {}
        for tag in ("warm", "timed"):
            vcf_path, snf_path = os.path.join(tmp, f"{tag}_{world}.vcf.gz"), os.path.join(tmp, f"{tag}_{world}.snf")
            cfg = sconfig.default_config("--input", bam, "--vcf", vcf_path, "--snf", snf_path, "--all-contigs", "--allow-overwrite",
                                         "--gpus", str(world))
            cfg.input = bam
            stats = {}
            tdist.barrier()
            t0 = time.perf_counter()
            n = call.call_sample(cfg, device=rank, stats=stats)
            wall = time.perf_counter() - t0
            out = {"wall_s": wall, "records_written": n, "stats": stats, "vcf": vcf_path, "snf": snf_path}
        if rank == 0:
            q.put(out)
    finally:
        tdist.destroy_process_group()


def run_size(bam, world, tmp):
    """call_sample at one world size on devices 0..world-1: rank 0's wall time, stats and output paths"""
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank, args=(r, world, port, bam, tmp, q)) for r in range(world)]
    for p in procs:
        p.start()
    try:
        out = q.get(timeout=3600)
        for p in procs:
            p.join(timeout=600)
        if any(p.exitcode != 0 for p in procs):
            raise RuntimeError(f"rank exit codes {[p.exitcode for p in procs]}")
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    return out


def summary(res, world):
    st = res["stats"]
    keys = ("tasks", "weight", "inflated_bytes", "passes", "index_s", "read_s", "load_bam_s", "run_s", "finalize_s", "vcf_write_s", "wall_s")
    if world == 1:
        ranks = [{k: st.get(k) for k in keys if k in st}]
        ranks[0]["inflated_bytes"] = sum(st["pass_inflated_bytes"])
    else:
        ranks = [{k: r.get(k) for k in keys} for r in st["ranks"]]
    for r in ranks:
        r["load_bam_s"], r["run_s"] = sum(r["load_bam_s"]), sum(r["run_s"])
    out = {"wall_s": res["wall_s"], "records_written": res["records_written"], "ranks": ranks}
    if world > 1:
        w = [r["weight"] for r in ranks]
        out["lpt_load_max_over_mean"] = max(w) / (sum(w) / len(w)) if sum(w) else None
        out["gather_s"], out["write_s"] = st["gather_s"], st["write_s"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", default="c6,c2")
    ap.add_argument("--c2-scale", type=float, default=0.01)
    ap.add_argument("--sizes", default="1,2,4,8")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("call_sample_scaling needs a CUDA device")
    import call_sample_bench as csb
    n_dev = torch.cuda.device_count()
    sizes = [n for n in map(int, a.sizes.split(",")) if n <= n_dev]
    out = {"card": csb.card(), "visible_devices": n_dev, "sizes": sizes, "inputs": {}}
    tmp = tempfile.mkdtemp(prefix="snfb_call_sample_scaling_")
    for kind in a.inputs.split(","):
        path, n_rec, bp = csb.make_input(kind, a.c2_scale, tmp)
        r = {"records": n_rec, "aligned_bp": bp, "bam_bytes": os.path.getsize(path), "by_size": {}}
        base = None
        for world in sizes:
            res = run_size(path, world, tmp)
            s = summary(res, world)
            s["sha256"] = files_sha256(res["vcf"], res["snf"])
            base = base or s["sha256"]
            s["same_files_as_one_rank"] = s["sha256"] == base
            r["by_size"][str(world)] = s
            print(f"[call_sample_scaling] {kind} x{world}: {json.dumps(s)}", file=sys.stderr, flush=True)
        out["inputs"][kind] = r
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
