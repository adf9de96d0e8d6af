"""Calling a whole sample from its BAM (`sniffles -i sample.bam -v out.vcf [--snf out.snf]`, the call_sample mode of sniffles:131-590).

  * planning is tasks.plan, shared with --genotype-vcf: one task per processed contig, [0, length - 1], task ids counted as the
    reference counts them; config.task_read_id_offset_mult follows sniffles:304-309 from the index's mapped-read counts;
  * the genome streams through the device in passes: consecutive tasks, in task-id order, whose inflated BAM bytes (the ISIZE of every
    BGZF block bamio.BamFile.device_input selects for them) fit a budget.  A pass is one mask_block, one snfb_load_bam and one snfb_run;
    its tasks then run as tasks.CallTask on the pass's BlockRun, and their VCF records and SNF parts are written before the next pass
    loads (host memory stays bounded, and snfb_coverage_bins reads the block loaded on the context);
  * the VCF goes through vcf.open_output (a .vcf.gz gets BGZF compressed on the GPU and a .tbi), the SNF through snf.write_results;
  * with --gpus N > 1, under torchrun, every rank runs its share of the tasks and rank 0 writes the files (call_sample_ranks)."""
import contextlib
import logging
import math
import os
import time

import numpy as np

from . import abi, bamio, binding, snf, tasks, vcf

log = logging.getLogger("sniffles_b200.call")

# Peak device memory of one snfb_load_bam + snfb_run, as measured with scripts/call_sample_bench.py on an H100 80GB HBM3 (700 W; DESIGN §8):
# 2.02 GB for 0.396 GB of inflated BAM (config 6) and 4.67 GB for 1.55 GB (config 2 at 1/100), i.e. about 1.1 GB fixed + 2.3 bytes per
# inflated byte.  The budget of a pass is the free device memory, less the fixed part, over the per-byte factor; both carry a margin.
DEVICE_BYTES_PER_INFLATED_BYTE = 2.6
DEVICE_BYTES_FIXED = 1_500_000_000
# the share of the free device memory a pass may plan on: the rest is left for the coverage bins, the REF gathers and the VCF compression
FREE_MEMORY_SHARE = 0.9


class CallSampleError(RuntimeError):
    """the run stops as the reference's util.fatal_error_main stops it; the message is the reference's where it has one"""


def read_id_offset_mult(total_mapped):
    """config.task_read_id_offset_mult (sniffles:304-309): 10 ** ceil(ln(total_mapped) + 1), 10 ** 9 when the index counts no mapped
    reads (the reference's CRAM case)"""
    if total_mapped == 0:
        return 10 ** 9
    return 10 ** math.ceil(math.log(total_mapped) + 1)


def total_mapped(bam):
    """pysam's AlignmentFile.mapped: the mapped-read counts of the index's pseudo-bins, summed over the contigs"""
    return sum(bam.count_mapped(name) or 0 for name, _ in bam.contigs)


def check_outputs(config):
    """the reference's checks before it opens any output (sniffles:122-127, 238-248, 265-267)"""
    if config.vcf is None and config.snf is None:
        raise CallSampleError("Please specify at least one of: --vcf or --snf for output (both may be used at the same time)")
    for path in (config.vcf, config.snf):
        if path is not None and os.path.exists(path) and not config.allow_overwrite:
            raise CallSampleError(f"Output file '{path}' already exists! Use --allow-overwrite to ignore this check and overwrite.")
    if config.vcf is not None:
        parent = os.path.dirname(os.path.abspath(config.vcf))
        if not os.path.exists(parent):
            raise CallSampleError(f"Directory {parent} does not exists.")


def inflated_bytes(bgzf):
    """the sum of ISIZE over whole BGZF members: what snfb_load_bam inflates them to"""
    return sum(isize for _, _, _, isize in bamio.bgzf_members(np.ascontiguousarray(bgzf, dtype="u1").tobytes()))


def device_budget(device=0):
    """the inflated BAM bytes one pass may load: the device's free memory, less DEVICE_BYTES_FIXED, over DEVICE_BYTES_PER_INFLATED_BYTE
    (at least one byte: a task larger than the budget still runs, alone in its pass)"""
    import torch
    free, _ = torch.cuda.mem_get_info(device)
    return max(1, int((free * FREE_MEMORY_SHARE - DEVICE_BYTES_FIXED) / DEVICE_BYTES_PER_INFLATED_BYTE))


def group_passes(items, budget, size=lambda item: item[-1]):
    """consecutive items, in order, grouped so that the sizes of a group sum to at most `budget`; an item larger than the budget forms a
    group of its own.  Lazy: an item is taken from `items` only when the group before it is complete or still has room."""
    group, used = [], 0
    for item in items:
        n = size(item)
        if group and used + n > budget:
            yield group
            group, used = [], 0
        group.append(item)
        used += n
    if group:
        yield group


def task_inputs(bam, planned, stats=None, regions_by_contig=None, failed=None):
    """per planned task, in task order: (task id, contig, start, end, BGZF bytes, spans, inflated bytes, regions) of
    bamio.BamFile.device_input over the task's fetch windows (tasks.fetch_windows; regions: those windows when the contig has regions, else
    None).  A task whose regions pysam would refuse is logged and left out, as the reference's worker fails it (and listed in `failed` as
    (task id, contig, error class name)).  The time spent reading is added to stats["read_s"]"""
    for tid, name, s, e in planned:
        t0 = time.perf_counter()
        rg = (regions_by_contig or {}).get(name)
        try:
            windows = tasks.fetch_windows(name, s, e, rg)
        except ValueError as err:
            log.error(f"Error in worker process while executing CallTask(id={tid}, contig={name}, start={s}, end={e}): {err}")
            if failed is not None:
                failed.append((tid, name, type(err).__name__))
            continue
        z, spans = bam.device_input([(name, a, b) for a, b in windows], tags=[(0, g) for g in range(len(windows))])
        n = inflated_bytes(z)
        if stats is not None:
            stats["read_s"] += time.perf_counter() - t0
        yield tid, name, s, e, z, spans, n, (windows if rg else None)


def join_inputs(inputs, n_regions=None):
    """the device_input of several tasks as one snfb_load_bam input: the BGZF bytes back to back, each task's spans shifted to its bytes
    and numbered by its place in the pass; n_regions: per task the number of its regions, whose span tags move to the pass's region table"""
    parts, rows, base, rbase = [], [], 0, 0
    for k, (z, spans) in enumerate(inputs):
        sp = spans.copy()
        sp["cbeg"] += base
        sp["cend"] += base
        sp["task"] = k
        if n_regions is not None:
            sp["region"] += rbase
            rbase += n_regions[k]
        parts.append(z)
        rows.append(sp)
        base += len(z)
    bgzf = np.concatenate(parts) if parts else np.zeros(0, "u1")
    return bgzf, np.concatenate(rows) if rows else np.zeros(0, abi.SPAN_DTYPE)


def load_pass(ctx, bam, group, config, tr_all, contigs=None, read_names=False):
    """the device half of a pass over `group` (items of task_inputs): mask_block, set_config, set_regions, snfb_load_bam and snfb_run,
    the k-th task of the group being task index k of the block.  Returns the pass's tasks.BlockRun and its split {"load_bam_s", "run_s"};
    a load or run the library refuses raises CallSampleError naming the pass's contigs and inflated bytes.  contigs: the names
    tasks.reference_for loads (None: all).  read_names: also gather the candidates' read names (snfb_read_names, before the next load
    replaces the records) into BlockRun.read_names, timed as split["rnames_s"]."""
    tr = {k: [(int(a), int(b)) for a, b in tr_all[g[1]]] for k, g in enumerate(group) if g[1] in tr_all}
    # a task with regions: its records carry their region's window, its own bounds only clip the N mask (the host clips it to the regions)
    bounds = [(0, bam.get_reference_length(name)) if rg else (s, e) for _, name, s, e, _, _, _, rg in group]
    block = bamio.pack_records(bam.contigs, [], [(bam.name_to_id[g[1]], a, b, g[0]) for g, (a, b) in zip(group, bounds)], tandem_repeats=tr or None)
    by_task = [(k, g[7] or [(g[2], g[3])]) for k, g in enumerate(group)]
    has_regions = any(g[7] for g in group)
    mask_regions = {k: g[7] for k, g in enumerate(group) if g[7]}
    # without regions or a contig subset the N mask is the plain mask_block(block, config, ctx), as --genotype-vcf has always called it
    tasks.mask_block(block, config, ctx, *((mask_regions or None, contigs) if mask_regions or contigs is not None else ()))
    ctx.set_config(abi.Config.from_sniffles(config))
    bgzf, spans = join_inputs([(g[4], g[5]) for g in group], [len(w) for _, w in by_task] if has_regions else None)
    split = {}
    try:
        t0 = time.perf_counter()
        ctx.set_regions(tasks.region_table(by_task) if has_regions else None)
        n_rec = ctx.load_bam(bgzf, spans, block)["n_rec"]
        t1 = time.perf_counter()
        res = ctx.run(want_leads=True, want_cands=True, want_seqs=True)
        t2 = time.perf_counter()
        names = tasks.read_names(ctx) if read_names else None
        t3 = time.perf_counter()
    except binding.SnfbError as e:
        contig_list = ", ".join(g[1] for g in group)
        raise CallSampleError(f"the device pass over contig(s) {contig_list} ({sum(g[6] for g in group)} inflated BAM bytes) failed: {e}") from e
    split["load_bam_s"], split["run_s"] = t1 - t0, t2 - t1
    if read_names:
        split["rnames_s"] = t3 - t2
    rec_nm = abi.view(res._rec_nm_ptr, "<f8", n_rec).copy() if getattr(res, "_rec_nm_ptr", None) else None
    return tasks.BlockRun(block, res, tasks.cand_ranges(res.cand, len(block.task)), rec_nm, read_names=names), split


def run_pass(ctx, bam, group, config, tr_all, device=0, contigs=None, failed=None):
    """one device pass over `group` (items of task_inputs): load_pass, then every task as a CallTask on the pass's BlockRun.  Returns
    [(CallTask, calls)] in task order and the pass's split {"load_bam_s", "run_s", "finalize_s"}, with --output-rnames also "rnames_s".
    contigs: the names tasks.reference_for loads (None: all); failed: receives (task id, contig, error class name) of every task that fails."""
    br, split = load_pass(ctx, bam, group, config, tr_all, contigs, read_names=bool(getattr(config, "output_rnames", False)))
    t2 = time.perf_counter()
    done = []
    for k, (tid, name, s, e, *_) in enumerate(group):
        task = tasks.CallTask(id=tid, sv_id=0, contig=name, start=s, end=e, config=config, block_run=br, task_index=k, device=device)
        try:
            calls, _ = task.execute()
        except tasks.CallTaskError as err:      # logged and left out, as the reference's worker leaves a failed task out
            log.error(f"Error in worker process while executing CallTask(id={tid}, contig={name}, start={s}, end={e}): {err}")
            if failed is not None:
                failed.append((tid, name, type(err).__name__))
            continue
        done.append((task, calls))
    split["finalize_s"] = time.perf_counter() - t2
    return done, split


def plan_sample(config):
    """what every run does before its first pass, the same on every rank: open config.input, set config.task_read_id_offset_mult,
    config.contig_lengths and config.sample_ids_vcf, plan the tasks and load the tandem repeats with the reference's fatal check.
    Returns (bam, processed contigs [(name, length)], planned tasks [(task id, name, start, end)], {contig: tandem repeats})."""
    path = config.input[0] if isinstance(config.input, (list, tuple)) else config.input
    bam = bamio.BamFile(path)
    config.task_read_id_offset_mult = read_id_offset_mult(total_mapped(bam))
    contig_lengths, planned = tasks.plan(bam.contigs, config)
    config.contig_lengths = contig_lengths
    tr_all = {}
    if config.tandem_repeats is not None:
        tr_all = tasks.load_tandem_repeats(config.tandem_repeats, config.tandem_repeat_region_pad)
        with_tr = sum(name in tr_all for name, _ in contig_lengths)
        if with_tr < len(contig_lengths):
            log.info(f"Info: {with_tr} of {len(contig_lengths)} contigs in the input sample have associated tandem repeat annotations.")
            if with_tr == 0:
                raise CallSampleError("A tandem repeat annotations file was provided, but no matching annotations were found for any contig in "
                                      "the sample input file. Please check if the contig naming scheme in the tandem repeat annotations "
                                      "matches with the one in the input sample file.")
    config.sample_ids_vcf = [(0, "SAMPLE" if config.sample_id is None else config.sample_id)]
    return bam, contig_lengths, planned, tr_all


def _world_size():
    """the size of the initialised torch.distributed process group, 1 without one"""
    try:
        import torch.distributed as tdist
    except ImportError:
        return 1
    return tdist.get_world_size() if tdist.is_available() and tdist.is_initialized() else 1


def call_sample(config, device=0, budget=None, stats=None):
    """the call_sample run mode: config.input (one indexed BAM) -> config.vcf and / or config.snf.  budget: the inflated BAM bytes one
    device pass may load (default: device_budget).  stats: a dict that receives the run's split (passes, per-pass inflated bytes and
    times, VCF and SNF write times).  Returns the number of VCF records written.

    With --gpus N > 1 the run is one process per GPU (torchrun --nproc-per-node N -m sniffles_b200 ... --gpus N): it needs an initialised
    process group of N ranks and goes through call_sample_ranks."""
    gpus = getattr(config, "gpus", 1)
    if gpus > 1:
        world = _world_size()
        if world == 1:
            raise CallSampleError(f"--gpus {gpus} runs one process per GPU: launch with torchrun --nproc-per-node {gpus} -m sniffles_b200 ... "
                                  f"--gpus {gpus}")
        if world != gpus:
            raise CallSampleError(f"--gpus {gpus} does not match the {world} ranks of the process group")
        return call_sample_ranks(config, device, budget, stats)
    check_outputs(config)
    st = stats if stats is not None else {}
    t0 = time.perf_counter()
    bam, contig_lengths, planned, tr_all = plan_sample(config)
    ctx = tasks.device_context(device)
    reference = tasks.reference_for(ctx, config.reference) if getattr(config, "reference", None) else None
    if budget is None:
        budget = device_budget(device)
    st.update(passes=0, pass_inflated_bytes=[], load_bam_s=[], run_s=[], rnames_s=[], finalize_s=0.0, vcf_write_s=0.0, snf_write_s=0.0, read_s=0.0)
    st["index_s"] = time.perf_counter() - t0
    parts, written = [], 0
    with contextlib.ExitStack() as stack:
        writer = None
        if config.vcf is not None:
            handle = vcf.open_output(config, ctx)
            if config.vcf_output_bgz:
                stack.enter_context(handle)               # compressed and indexed when the run ends without an error
            else:
                stack.callback(handle.close)
            writer = vcf.VCFWriter(config, handle, reference)
            writer.write_header(contig_lengths)
        for group in group_passes(task_inputs(bam, planned, st, config.regions_by_contig), budget, size=lambda item: item[6]):
            done, split = run_pass(ctx, bam, group, config, tr_all, device)
            st["passes"] += 1
            st["pass_inflated_bytes"].append(sum(g[6] for g in group))
            st["load_bam_s"].append(split["load_bam_s"])
            st["run_s"].append(split["run_s"])
            if "rnames_s" in split:
                st["rnames_s"].append(split["rnames_s"])
            st["finalize_s"] += split["finalize_s"]
            t1 = time.perf_counter()
            if writer is not None:
                if reference is not None:
                    reference.prefetch(vcf.reference_intervals([c for _, calls in done for c in calls], config))
                for _, calls in done:
                    for c in calls:
                        written += writer.write_call(c)
            t2 = time.perf_counter()
            parts.extend(task.snf_part for task, _ in done if task.snf_part is not None)
            st["vcf_write_s"] += t2 - t1
        t1 = time.perf_counter()
    st["vcf_write_s"] += time.perf_counter() - t1          # the .vcf.gz compression and .tbi when the handle closes
    if config.snf is not None:
        t1 = time.perf_counter()
        with open(config.snf, "wb") as f:
            n = snf.write_results(f, config, parts, [name for name, _ in contig_lengths])
        st["snf_write_s"] = time.perf_counter() - t1
        log.info(f"Wrote {n} SV candidates to {config.snf} (for multi-sample calling).")
    if config.vcf is not None:
        log.info(f"Wrote {written} called SVs to {config.vcf}")
    st["wall_s"] = time.perf_counter() - t0
    return written


def run_rank_tasks(config, device, budget, rank, world):
    """one rank's share of a multi-GPU run: the plan every rank makes alike (plan_sample), the tasks dist.lpt_assign gives this rank over
    dist.task_weights, then the loop of call_sample over them in task-id order, each task's VCF records formatted here into text.  With
    --reference only the contigs of this rank's tasks are loaded, and the N mask and the VCF writer use that one object.  Returns the
    payload rank 0 merges (write_rank_outputs): {"rank", "tasks": [(task id, VCF text, records, SNF part or None)], "failed": [(task id,
    contig, error class name)], "nm": (last task id, average_regional_nm, qc_nm_threshold) or None, "stats", "error": None}."""
    import io
    from . import dist
    t0 = time.perf_counter()
    st = dict(passes=0, pass_inflated_bytes=[], load_bam_s=[], run_s=[], rnames_s=[], finalize_s=0.0, vcf_write_s=0.0, read_s=0.0)
    bam, contig_lengths, planned, tr_all = plan_sample(config)
    weights = dist.task_weights(bam, planned, config.regions_by_contig)
    owner = dist.lpt_assign(weights, world)
    mine = [p for p, o in zip(planned, owner) if o == rank]
    contigs = sorted({name for _, name, _, _ in mine})
    ctx = tasks.device_context(device)
    reference = tasks.reference_for(ctx, config.reference, contigs) if getattr(config, "reference", None) and mine else None
    if budget is None:
        budget = device_budget(device)
    st.update(tasks=len(mine), weight=sum(w for w, o in zip(weights, owner) if o == rank), index_s=time.perf_counter() - t0)
    out, failed, nm = [], [], None
    for group in group_passes(task_inputs(bam, mine, st, config.regions_by_contig, failed), budget, size=lambda item: item[6]):
        done, split = run_pass(ctx, bam, group, config, tr_all, device, contigs, failed)
        # the config holds the N-mismatch mean of the pass's last task: the SNF header of rank 0 takes that of the run's last task
        nm = (group[-1][0], config.average_regional_nm, config.qc_nm_threshold)
        st["passes"] += 1
        st["pass_inflated_bytes"].append(sum(g[6] for g in group))
        st["load_bam_s"].append(split["load_bam_s"])
        st["run_s"].append(split["run_s"])
        if "rnames_s" in split:
            st["rnames_s"].append(split["rnames_s"])
        st["finalize_s"] += split["finalize_s"]
        t1 = time.perf_counter()
        if config.vcf is not None and reference is not None:
            reference.prefetch(vcf.reference_intervals([c for _, calls in done for c in calls], config))
        for task, calls in done:
            text, n = "", 0
            if config.vcf is not None:
                buf = io.StringIO()
                writer = vcf.VCFWriter(config, buf, reference)
                n = sum(writer.write_call(c) for c in calls)
                text = buf.getvalue()
            out.append((task.id, text, n, task.snf_part))
        st["vcf_write_s"] += time.perf_counter() - t1
    bam.close()
    st["inflated_bytes"] = sum(st["pass_inflated_bytes"])
    st["wall_s"] = time.perf_counter() - t0
    return {"rank": rank, "tasks": out, "failed": failed, "nm": nm, "stats": st, "error": None}


def write_rank_outputs(config, contig_lengths, payloads, ctx=None):
    """rank 0's merge of every rank's payload (run_rank_tasks): when any rank failed, no file is written and CallSampleError names the
    first failed rank and its message; otherwise the VCF header, then every task's records in task-id
    order through vcf.open_output (a .vcf.gz compressed on the device of `ctx`), and the SNF through snf.write_results.  Returns (records
    written, VCF write seconds, SNF write seconds)."""
    failed = [p for p in payloads if p["error"] is not None]
    if failed:
        raise CallSampleError(f"rank {failed[0]['rank']}: {failed[0]['error']}")
    done = sorted((t for p in payloads for t in p["tasks"]), key=lambda t: t[0])
    last = max((p["nm"] for p in payloads if p["nm"] is not None), default=None, key=lambda x: x[0])
    if last is not None:
        config.average_regional_nm, config.qc_nm_threshold = last[1], last[2]
    written, vcf_s, snf_s = 0, 0.0, 0.0
    if config.vcf is not None:
        t0 = time.perf_counter()
        with contextlib.ExitStack() as stack:
            handle = vcf.open_output(config, ctx)
            if config.vcf_output_bgz:
                stack.enter_context(handle)           # compressed and indexed when the writing ends without an error
            else:
                stack.callback(handle.close)
            vcf.VCFWriter(config, handle).write_header(contig_lengths)
            for _, text, n, _ in done:
                handle.write(text)
                written += n
        vcf_s = time.perf_counter() - t0
    if config.snf is not None:
        t0 = time.perf_counter()
        with open(config.snf, "wb") as f:
            n = snf.write_results(f, config, [t[3] for t in done if t[3] is not None], [name for name, _ in contig_lengths])
        snf_s = time.perf_counter() - t0
        log.info(f"Wrote {n} SV candidates to {config.snf} (for multi-sample calling).")
    if config.vcf is not None:
        log.info(f"Wrote {written} called SVs to {config.vcf}")
    return written, vcf_s, snf_s


def _error_text(e):
    return str(e) if isinstance(e, CallSampleError) else f"{type(e).__name__}: {e}"


def call_sample_ranks(config, device, budget=None, stats=None):
    """call_sample over the ranks of an initialised torch.distributed process group (one process per GPU; gloo, since the only
    collectives carry host objects).  Rank 0 checks the outputs and broadcasts the verdict; every rank plans alike, runs its own tasks
    (run_rank_tasks) and sends its payload to rank 0 with gather_object, an error included, so that every rank reaches the gather.  Rank 0
    writes the files (write_rank_outputs) and broadcasts (ok, records written or the error): every rank returns the same count or raises
    the same CallSampleError.  Rank 0 holds every rank's VCF text and SNF parts at once, host memory in proportion to the output files.

    stats on rank 0: the keys of call_sample for rank 0's own work, plus "ranks" (per rank its split, tasks, inflated bytes, index weight
    and failed tasks), "gather_s" and "write_s"."""
    import torch.distributed as tdist
    rank, world = tdist.get_rank(), tdist.get_world_size()
    t0 = time.perf_counter()
    verdict = [None]
    if rank == 0:
        try:
            check_outputs(config)
        except CallSampleError as e:
            verdict[0] = str(e)
    tdist.broadcast_object_list(verdict, src=0)
    if verdict[0] is not None:
        raise CallSampleError(verdict[0])
    try:
        payload = run_rank_tasks(config, device, budget, rank, world)
    except Exception as e:                   # into the payload: a rank that raised before the gather would leave the others waiting
        log.error(_error_text(e))
        payload = {"rank": rank, "tasks": [], "failed": [], "nm": None, "stats": {}, "error": _error_text(e)}
    t1 = time.perf_counter()
    gathered = [None] * world if rank == 0 else None
    tdist.gather_object(payload, gathered, dst=0)
    status = [None]
    if rank == 0:
        t2 = time.perf_counter()
        try:
            written, vcf_s, snf_s = write_rank_outputs(config, getattr(config, "contig_lengths", []), gathered, tasks.device_context(device))
            status[0] = (True, written)
        except Exception as e:
            status[0] = (False, _error_text(e))
        t3 = time.perf_counter()
        if status[0][0] and stats is not None:
            stats.update({k: v for k, v in payload["stats"].items() if k not in ("tasks", "weight", "inflated_bytes")})
            stats["vcf_write_s"] += vcf_s
            stats["snf_write_s"] = snf_s
            stats["ranks"] = [dict(p["stats"], failed=p["failed"]) for p in gathered]
            stats["gather_s"], stats["write_s"] = t2 - t1, t3 - t2
            stats["wall_s"] = t3 - t0
    tdist.broadcast_object_list(status, src=0)
    ok, value = status[0]
    if not ok:
        raise CallSampleError(value)
    return value
