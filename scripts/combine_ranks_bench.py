"""Combine mode on several ranks: combine_sample_bench's 50-sample cohort written once, then combine_run.combine_snfs over it at world
sizes 1, 2, 4 and 8 (capped at the visible devices; with --share-device every rank runs on device 0, a measure of the host decode spread
over processes, not of several GPUs).  Each world size is one gloo group of spawned processes, one per rank; the timed window starts after
a barrier that follows every rank's device context creation.  Prints the card's name and power limit, then one JSON line per world size:
the wall time, per rank decode_s / device_s / call_group_s / write_s (formatting its records, and at world size 1 writing the file),
task count and SNF-byte weight, gather_s and merge_write_s of rank 0's merge (null at world size 1), the records and dropped calls, and
whether the file is byte-equal to world size 1's.

    python scripts/combine_ranks_bench.py [--scale 0.1] [--share-device] [--worlds 1,2,4,8]"""
import argparse
import datetime
import hashlib
import json
import multiprocessing as mp
import os
import queue
import socket
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def _rank(rank, world, port, device, paths, vcf_path, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      LOCAL_WORLD_SIZE=str(world))
    import torch
    import torch.distributed as tdist
    from sniffles_b200 import combine_run, tasks
    from sniffles_b200 import config as sconfig
    torch.cuda.set_device(device)
    tasks.device_context(device)                                 # context creation outside the timed window
    if world > 1:
        tdist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(hours=1))
        tdist.barrier()
    try:
        cfg = sconfig.SnifflesConfig("-i", *paths, "-v", vcf_path, "--allow-overwrite", "--gpus", str(world))
        cfg.command, cfg.start_date = "sniffles combine_ranks_bench", "2026/01/01 00:00:00"
        st = {}
        t0 = time.perf_counter()
        n = combine_run.combine_snfs(cfg, device=device, stats=st)
        wall = time.perf_counter() - t0
        q.put((rank, True, {"n": n, "wall_s": wall, "stats": st}))
    except Exception as e:
        q.put((rank, False, f"{type(e).__name__}: {e}"))
    finally:
        if world > 1:
            tdist.destroy_process_group()


def run_world(world, devices, paths, vcf_path, timeout=3600):
    """rank 0's result of one combine over `world` spawned ranks on `devices`; every rank is joined or terminated before it returns"""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    procs = [ctx.Process(target=_rank, args=(r, world, port, devices[r], paths, vcf_path, q)) for r in range(world)]
    for p in procs:
        p.start()
    got, deadline = {}, time.monotonic() + timeout
    try:
        while len(got) < world:
            try:
                rank, ok, value = q.get(timeout=max(1.0, deadline - time.monotonic()))
            except queue.Empty:
                raise SystemExit(f"world {world}: ranks {sorted(set(range(world)) - set(got))} did not report within {timeout} s") from None
            if not ok:
                raise SystemExit(f"world {world}, rank {rank}: {value}")
            got[rank] = value
        for p in procs:
            p.join(timeout=max(1.0, deadline - time.monotonic()))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    return got[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--share-device", action="store_true", help="every rank on device 0")
    ap.add_argument("--worlds", default="1,2,4,8")
    args = ap.parse_args()
    import torch
    import combine_sample_bench
    n_dev = torch.cuda.device_count()
    if n_dev == 0:
        raise SystemExit("combine_ranks_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    worlds = [w for w in (int(x) for x in args.worlds.split(",")) if args.share_device or w <= n_dev]
    print(json.dumps({"gpu": gpu, "visible_devices": n_dev, "share_device": args.share_device, "worlds": worlds,
                      "workload": f"combine_sample_bench cohort: 50 samples, scale {args.scale}"}), flush=True)
    with tempfile.TemporaryDirectory() as tmp:
        paths = combine_sample_bench.write_cohort(tmp, args.scale)
        digest1 = None
        for world in worlds:
            vcf_path = os.path.join(tmp, f"w{world}.vcf")
            devices = [0] * world if args.share_device else list(range(world))
            res = run_world(world, devices, paths, vcf_path)
            with open(vcf_path, "rb") as f:
                digest = hashlib.sha256(f.read()).hexdigest()
            if digest1 is None and world == 1:
                digest1 = digest
            st = res["stats"]
            ranks = st.get("ranks") or [st]
            print(json.dumps({"world": world, "wall_s": round(res["wall_s"], 3), "records": res["n"], "dropped": st["dropped"],
                              "ranks": [{k: (round(r[k], 3) if isinstance(r.get(k), float) else r.get(k)) for k in ("decode_s", "device_s", "call_group_s", "write_s", "tasks", "weight")}
                                        for r in ranks],
                              "gather_s": round(st["gather_s"], 3) if world > 1 else None,
                              "merge_write_s": round(st["write_s"], 3) if world > 1 else None,
                              "equal_to_world_1": None if digest1 is None else digest == digest1}), flush=True)


if __name__ == "__main__":
    main()
