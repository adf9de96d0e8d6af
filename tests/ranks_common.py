"""Several ranks of a torch.distributed gloo group as spawned processes on this host, for the tests of call.call_sample_ranks and of the
command line under a world size > 1.  Every process is joined with a deadline and terminated when the run fails or times out, so no
rank outlives the test."""
import datetime
import multiprocessing as mp
import os
import queue
import socket
import time


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_main(fn, rank, world, port, init, q, args):
    """one spawned rank: torchrun's environment, the gloo group when `init`, then fn(rank, world, *args) -> (rank, ok, value or error)"""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank),
                      LOCAL_WORLD_SIZE=str(world))
    import torch.distributed as tdist
    if init:
        tdist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=300))
    try:
        out = (rank, True, fn(rank, world, *args))
    except Exception as e:
        out = (rank, False, f"{type(e).__name__}: {e}")
    finally:
        if init:
            tdist.destroy_process_group()
    q.put(out)


def run_ranks(fn, world, *args, init=True, timeout=600):
    """fn(rank, world, *args) on `world` spawned ranks (fn: a module-level function).  Returns [(ok, value or error text)] in rank order;
    raises when a rank does not report or exit in time, after terminating every rank still alive."""
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_rank_main, args=(fn, r, world, port, init, q, args)) for r in range(world)]
    for p in procs:
        p.start()
    deadline = time.monotonic() + timeout
    got = {}
    try:
        while len(got) < world:
            try:
                rank, ok, value = q.get(timeout=max(1.0, deadline - time.monotonic()))
            except queue.Empty:
                raise TimeoutError(f"ranks {sorted(set(range(world)) - set(got))} did not report within {timeout} s") from None
            got[rank] = (ok, value)
        for p in procs:
            p.join(timeout=max(1.0, deadline - time.monotonic()))
        codes = [p.exitcode for p in procs]
        if codes != [0] * world:
            raise RuntimeError(f"rank exit codes {codes}")
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
    return [got[r] for r in range(world)]
