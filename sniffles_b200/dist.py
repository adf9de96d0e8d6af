"""Multi-GPU plumbing (SURVEY.md §8e): the path shards by contig — one process per GPU, contigs
assigned longest-first, no data-path collective — and ends with ONE all-gather that concatenates
the per-rank candidate buffers before VCF emission.  torch.distributed is used for the
collective only (NCCL over NVLink on the GPU box, gloo in the CPU tests).

Calling a sample on several GPUs (call.call_sample_ranks) weighs its tasks with task_weights,
assigns them with lpt_assign, and gathers each rank's finished VCF text and SNF parts instead.  Combining samples on several GPUs
(combine_run.combine_snfs_ranks) weighs its combine tasks with combine_task_weights.  Both run through rank_run."""
import bisect
import os
import time

import numpy as np


def lpt_assign(weights, n_ranks):
    """contig -> rank, longest-processing-time first.  The reference's unit of parallelism is the contig
    (sniffles:313-358); clusters never cross a task, so any contig partition gives identical calls."""
    load = [0] * n_ranks
    owner = [0] * len(weights)
    for c in sorted(range(len(weights)), key=lambda k: (-weights[k], k)):
        r = min(range(n_ranks), key=lambda k: (load[k], k))
        owner[c] = r
        load[r] += weights[c]
    return owner


def _block_bounds(bam):
    """the BGZF block starts the BAM index names (every chunk bound, linear-index entry and CSI loffset), and the file's end, sorted"""
    starts = {os.path.getsize(bam.path)}
    for bins, lin, loff in bam.index:
        for b, chunks in bins.items():
            if b != bam.meta_bin:                    # the pseudo-bin holds counts, not offsets
                starts.update(v >> 16 for c in chunks for v in c)
        starts.update(v >> 16 for v in (lin or ()))
        starts.update(v >> 16 for v in (loff or {}).values())
    return sorted(starts)


def task_weights(bam, planned, regions_by_contig=None):
    """per planned task [(task id, contig, start, end)] of tasks.plan, the compressed BAM bytes its fetches read: the BGZF blocks of
    every bamio.BamFile.merged_chunks range over the task's tasks.fetch_windows.  Read from the index alone, so a rank that weighs the
    tasks reads no BGZF block: a range that ends inside a block counts that block up to the next block start the index names.  A task
    whose windows are refused weighs 0: it fails on whichever rank runs it."""
    from . import tasks
    bounds = _block_bounds(bam)

    def chunk_bytes(vb, ve):
        cb, ce = vb >> 16, ve >> 16
        if ve & 0xffff:
            ce = bounds[min(bisect.bisect_right(bounds, ce), len(bounds) - 1)]
        return max(ce - cb, 0)

    out = []
    for _, name, s, e in planned:
        try:
            windows = tasks.fetch_windows(name, s, e, (regions_by_contig or {}).get(name))
        except ValueError:
            out.append(0)
            continue
        out.append(sum(chunk_bytes(vb, ve) for a, b in windows for vb, ve in bam.merged_chunks(name, a, b)))
    return out


def combine_task_weights(readers, planned):
    """per planned combine.CombineTask, the compressed SNF bytes of its blocks summed over every sample: the lengths of the parts each
    SNFReader.index ({contig: {str(block): [(offset, length), ...]}}) lists for the task's block_indices.  Read from the headers alone:
    no block is decoded.  readers: {internal id: snf.SNFReader}"""
    out = []
    for task in planned:
        w = 0
        for r in readers.values():
            blocks = r.index.get(task.contig, {})
            w += sum(length for b in task.block_indices for _, length in blocks.get(str(b), ()))
        out.append(w)
    return out


def rank_run(check, work, write, error, log, failed_payload, timing=None):
    """One run over the ranks of an initialised torch.distributed process group (one process per GPU; gloo, since the only collectives
    carry host objects).  Rank 0 alone runs check() and broadcasts its verdict (an `error` raised there stops every rank with its
    message).  Every rank then runs work(rank, world) -> its payload; an exception is logged and caught into failed_payload(rank, text), so
    that every rank reaches the gather.  gather_object brings the payloads, in rank order, to rank 0, which runs write(payloads) and
    broadcasts (ok, its value or the error): every rank returns the same value or raises the same `error`.

    timing: a dict that receives, on rank 0 when the write succeeds, gather_s (from the end of its own work to the end of the gather),
    write_s and wall_s."""
    import torch.distributed as tdist

    def text(e):
        return str(e) if isinstance(e, error) else f"{type(e).__name__}: {e}"

    rank, world = tdist.get_rank(), tdist.get_world_size()
    t0 = time.perf_counter()
    verdict = [None]
    if rank == 0:
        try:
            check()
        except error as e:
            verdict[0] = str(e)
    tdist.broadcast_object_list(verdict, src=0)
    if verdict[0] is not None:
        raise error(verdict[0])
    try:
        payload = work(rank, world)
    except Exception as e:                   # into the payload: a rank that raised before the gather would leave the others waiting
        log.error(text(e))
        payload = failed_payload(rank, text(e))
    t1 = time.perf_counter()
    gathered = [None] * world if rank == 0 else None
    tdist.gather_object(payload, gathered, dst=0)
    status = [None]
    if rank == 0:
        t2 = time.perf_counter()
        try:
            status[0] = (True, write(gathered))
        except Exception as e:
            status[0] = (False, text(e))
        t3 = time.perf_counter()
        if status[0][0] and timing is not None:
            timing.update(gather_s=t2 - t1, write_s=t3 - t2, wall_s=t3 - t0)
    tdist.broadcast_object_list(status, src=0)
    ok, value = status[0]
    if not ok:
        raise error(value)
    return value


def subset_block(block, task_ids):
    """The records of the given tasks as a block of their own (arenas are shared, offsets stay valid; the parent's owner,
    reference N mask and CIGAR16 twin are carried along)."""
    keep = np.isin(block.rec["task"], np.asarray(sorted(task_ids), dtype=block.rec["task"].dtype))
    sub = type(block)(rec=np.ascontiguousarray(block.rec[keep]), cigar=block.cigar, var=block.var, seq=block.seq, task=block.task,
                      contig=block.contig, tr=block.tr, contig_names=block.contig_names, sites=block.sites, _owner=block._owner,
                      mask=block.mask, mask_task_off=block.mask_task_off)
    if block.cigar16 is not None:
        sub.rec16, sub.cigar16 = np.ascontiguousarray(block.rec16[keep]), block.cigar16
    return sub


def rank_reference(path, ctx, block, task_ids):
    """the reference FASTA of --reference loaded on a rank's device with only the contigs of its tasks (fasta.Reference); the N mask
    built from it travels with the block (subset_block)"""
    from . import fasta
    names = sorted({block.contig_names[int(block.task[t]["contig"])] for t in task_ids})
    return fasta.Reference(path, ctx, contigs=names)


def allgather_bytes(local, group=None):
    """All-gather of variable-length uint8 tensors: sizes first, then max-padded payloads.  Returns the list of
    per-rank tensors (trimmed).  `local` lives on the device of the backend (cuda for nccl, cpu for gloo)."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    n = torch.tensor([local.numel()], dtype=torch.int64, device=local.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n, group=group)
    sizes = [int(s.item()) for s in sizes]
    mx = max(max(sizes), 1)
    pad = torch.zeros(mx, dtype=torch.uint8, device=local.device)
    pad[:local.numel()] = local
    outs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad, group=group)
    return [o[:s] for o, s in zip(outs, sizes)]


def gather_struct_arrays(arr, group=None, device="cpu"):
    """All-gather a numpy structured array (e.g. snfb_cand records); returns the per-rank arrays."""
    import torch
    raw = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    t = torch.from_numpy(raw.copy()).to(device)
    parts = allgather_bytes(t, group)
    return [np.frombuffer(p.cpu().numpy().tobytes(), dtype=arr.dtype) for p in parts]


class DeviceBytes:
    """zero-copy view of a library-owned device buffer for torch (``torch.as_tensor(DeviceBytes(p, n), device='cuda')``)"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (int(nbytes),), "typestr": "|u1", "data": (int(ptr), False), "version": 3}


def merge_results(parts):
    """Host restatement of the library's k_gather_merge (csrc/api.cu): concatenate per-rank results in rank order and rebase
    alt_off / lead_off / long_off and the rnames offsets into the merged arenas.  parts: objects with cand, alt, rnames, rn_off,
    cand_leads (binding.Result / OracleResult).  Returns a binding.GatheredResult."""
    from .binding import GatheredResult
    from . import abi
    g = GatheredResult()
    cands, alts, rns, offs, leads = [], [], [], [], []
    b_alt = b_rn = b_leads = 0
    for p in parts:
        c = np.array(p.cand, copy=True)
        c["alt_off"] = np.where(c["alt_off"] >= 0, c["alt_off"] + b_alt, c["alt_off"])
        c["lead_off"] += b_leads
        c["long_off"] += b_leads
        cands.append(c)
        alts.append(np.asarray(p.alt, dtype="u1"))
        rns.append(np.asarray(p.rnames, dtype="<u8"))
        offs.append(np.asarray(p.rn_off[:len(c)], dtype="<u4") + np.uint32(b_rn))
        leads.append(np.asarray(p.cand_leads))
        b_alt += len(p.alt)
        b_rn += len(p.rnames)
        b_leads += len(p.cand_leads)
    g.cand = np.concatenate(cands) if cands else np.zeros(0, abi.CAND_DTYPE)
    g.alt = np.concatenate(alts) if alts else np.zeros(0, "u1")
    g.rnames = np.concatenate(rns) if rns else np.zeros(0, "<u8")
    g.rn_off = np.concatenate(offs + [np.asarray([b_rn], dtype="<u4")])
    g.cand_leads = np.concatenate(leads) if leads else np.zeros(0, abi.LEAD_DTYPE)
    g.n_cand, g.n_alt_bytes, g.n_rnames, g.n_cand_leads = len(g.cand), len(g.alt), len(g.rnames), len(g.cand_leads)
    return g


class _Part:
    pass


def gather_results(res, group=None, device="cpu"):
    """All-gather a rank's whole result (candidate records, ALT arena, read names + offsets, candidate leads) through
    torch.distributed and merge it (gloo on CPU: the test of the N > 1 host logic; the GPU path uses the library's own
    NCCL all-gather, snfb_allgather_candidates)."""
    from . import abi
    parts = None
    for name, dt in (("cand", abi.CAND_DTYPE), ("alt", np.dtype("u1")), ("rnames", np.dtype("<u8")), ("rn_off", np.dtype("<u4")), ("cand_leads", abi.LEAD_DTYPE)):
        arr = np.ascontiguousarray(getattr(res, name))
        got = gather_struct_arrays(arr.view(dt) if arr.dtype != dt else arr, group, device)
        if parts is None:
            parts = [_Part() for _ in got]
        for p, a in zip(parts, got):
            setattr(p, name, a)
    return merge_results(parts)


def merge_rank_candidates(parts):
    """Concatenate per-rank candidate arrays in reference emission order: task id, then each rank's own order
    (sniffles:544-547 sorts finished tasks by id).  Records only: use merge_results for the arenas."""
    allc = np.concatenate(parts) if parts else parts
    return allc[np.argsort(allc["task"], kind="stable")]
