"""Calling a whole sample from its BAM (`sniffles -i sample.bam -v out.vcf [--snf out.snf]`, the call_sample mode of sniffles:131-590).

  * planning is tasks.plan, shared with --genotype-vcf: one task per processed contig, [0, length - 1], task ids counted as the
    reference counts them; config.task_read_id_offset_mult follows sniffles:304-309 from the index's mapped-read counts;
  * the genome streams through the device in passes (device_passes, shared with --genotype-vcf): consecutive tasks, in task-id order,
    whose inflated BAM bytes (the ISIZE of every BGZF block bamio.BamFile.device_input selects for them) fit a budget.  A pass is
    tasks.pass_block (tables and N mask) and tasks.load_and_run (one snfb_load_bam and one snfb_run); its tasks then run as tasks.CallTask
    on the pass's BlockRun (run_pass), and their VCF records and SNF parts are written before the next pass loads (host memory stays
    bounded, and snfb_coverage_bins reads the block loaded on the context);
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


def open_indexed(path):
    """bamio.BamFile over `path` and its index; CallSampleError with the reference's message (sniffles:171-178) when there is no index"""
    if bamio.find_index(path) is None:
        raise CallSampleError(f"Unable to load index for input file '{path}'. Please verify that your input file is sorted + indexed and that the "
                              f"index .bai file is valid and in the right location. Build one on the GPU with: python -m sniffles_b200.index {path}")
    return bamio.BamFile(path)


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
    """per planned task, in task order, its tasks.TaskInput: bamio.BamFile.device_input over the task's fetch windows
    (tasks.fetch_windows), their inflated bytes, and the windows when the contig has regions.  A task whose regions pysam would refuse is
    logged and left out, as the reference's worker fails it (and listed in `failed`).  The time spent reading is added to
    stats["read_s"]"""
    for tid, name, s, e in planned:
        t0 = time.perf_counter()
        rg = (regions_by_contig or {}).get(name)
        try:
            windows = tasks.fetch_windows(name, s, e, rg)
        except ValueError as err:
            tasks.CallTask(tid, 0, name, s, e, None).log_failure(log, err, failed)
            continue
        z, spans = bam.device_input([(name, a, b) for a, b in windows], tags=[(0, g) for g in range(len(windows))])
        n = inflated_bytes(z)
        if stats is not None:
            stats["read_s"] += time.perf_counter() - t0
        yield tasks.TaskInput(tid, name, s, e, z, spans, n, windows if rg else None)


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


def load_pass(ctx, bam, group, config, tr_all, contigs=None):
    """the device half of a pass over `group` (TaskInputs of task_inputs, the k-th being task index k of the block): tasks.pass_block,
    then tasks.load_and_run over the tasks' joined BGZF bytes.  Returns the pass's tasks.BlockRun and its split; a load or run the library
    refuses raises CallSampleError naming the pass's contigs and inflated bytes.  contigs: the names tasks.reference_for loads (None: all)."""
    block = tasks.pass_block(ctx, bam, group, config, tr_all, contigs)
    has_regions = any(it.regions for it in group)
    windows = [(k, it.regions or [(it.start, it.end)]) for k, it in enumerate(group)] if has_regions else None
    bgzf, spans = join_inputs([(it.bgzf, it.spans) for it in group], [len(w) for _, w in windows] if has_regions else None)
    try:
        return tasks.load_and_run(ctx, config, block, windows, bgzf, spans)
    except binding.SnfbError as e:
        contig_list = ", ".join(it.contig for it in group)
        raise CallSampleError(f"the device pass over contig(s) {contig_list} ({sum(it.inflated for it in group)} inflated BAM bytes) failed: {e}") from e


def device_passes(ctx, bam, planned, config, tr_all, budget, stats, contigs=None, failed=None):
    """the device passes of a run over `planned` (task id, contig, start, end): the TaskInputs of task_inputs, grouped by group_passes
    under `budget` and run by load_pass, one pass at a time.  Yields (group, BlockRun); the next pass loads only when the caller asks for
    it, so everything the caller does with a pass sees its block on the context.  stats: receives read_s, passes, pass_inflated_bytes and
    per pass load_bam_s, run_s and, with --output-rnames, rnames_s.  contigs: as load_pass; failed: as task_inputs."""
    for group in group_passes(task_inputs(bam, planned, stats, config.regions_by_contig, failed), budget, size=lambda it: it.inflated):
        br, split = load_pass(ctx, bam, group, config, tr_all, contigs)
        stats["passes"] += 1
        stats["pass_inflated_bytes"].append(sum(it.inflated for it in group))
        for k in ("load_bam_s", "run_s", "rnames_s"):
            if k in split:
                stats.setdefault(k, []).append(split[k])
        yield group, br


def run_pass(group, br, config, device, stats, failed=None):
    """every task of a pass (`group`, run as `br` by device_passes) as a CallTask on the pass's BlockRun: [(CallTask, calls)] in task
    order, the time added to stats["finalize_s"].  failed: receives (task id, contig, error class name) of every task that fails."""
    t0 = time.perf_counter()
    done = []
    for k, it in enumerate(group):
        task = tasks.CallTask(id=it.id, sv_id=0, contig=it.contig, start=it.start, end=it.end, config=config, block_run=br, task_index=k, device=device)
        try:
            calls, _ = task.execute()
        except tasks.CallTaskError as err:      # logged and left out, as the reference's worker leaves a failed task out
            task.log_failure(log, err, failed)
            continue
        done.append((task, calls))
    stats["finalize_s"] += time.perf_counter() - t0
    return done


def plan_sample(config):
    """what every run does before its first pass, the same on every rank: open config.input, set config.task_read_id_offset_mult,
    config.contig_lengths and config.sample_ids_vcf, plan the tasks and load the tandem repeats with the reference's fatal check.
    Returns (bam, processed contigs [(name, length)], planned tasks [(task id, name, start, end)], {contig: tandem repeats})."""
    path = config.input[0] if isinstance(config.input, (list, tuple)) else config.input
    bam = open_indexed(path)
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
    # a .vcf.gz is compressed and indexed when the run ends without an error
    with vcf.open_output(config, ctx) if config.vcf is not None else contextlib.nullcontext() as handle:
        writer = None
        if handle is not None:
            writer = vcf.VCFWriter(config, handle, reference)
            writer.write_header(contig_lengths)
        for group, br in device_passes(ctx, bam, planned, config, tr_all, budget, st):
            done = run_pass(group, br, config, device, st)
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
    for group, br in device_passes(ctx, bam, mine, config, tr_all, budget, st, contigs, failed):
        done = run_pass(group, br, config, device, st, failed)
        # the config holds the N-mismatch mean of the pass's last task: the SNF header of rank 0 takes that of the run's last task
        nm = (group[-1].id, config.average_regional_nm, config.qc_nm_threshold)
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
        with vcf.open_output(config, ctx) as handle:          # a .vcf.gz is compressed and indexed when the writing ends without an error
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


def call_sample_ranks(config, device, budget=None, stats=None):
    """call_sample over the ranks of an initialised torch.distributed process group, through dist.rank_run: rank 0 checks the outputs
    and broadcasts the verdict; every rank plans alike, runs its own tasks (run_rank_tasks) and sends its payload to rank 0, an error
    included.  Rank 0 writes the files (write_rank_outputs): every rank returns the same count or raises the same CallSampleError.  Rank 0
    holds every rank's VCF text and SNF parts at once, host memory in proportion to the output files.

    stats on rank 0: the keys of call_sample for rank 0's own work, plus "ranks" (per rank its split, tasks, inflated bytes, index weight
    and failed tasks), "gather_s" and "write_s"."""
    from . import dist
    timing, merged = {}, {}

    def write(gathered):
        written, merged["vcf_s"], merged["snf_s"] = write_rank_outputs(config, getattr(config, "contig_lengths", []), gathered,
                                                                       tasks.device_context(device))
        merged["gathered"] = gathered
        return written

    written = dist.rank_run(lambda: check_outputs(config), lambda rank, world: run_rank_tasks(config, device, budget, rank, world), write,
                            CallSampleError, log,
                            lambda rank, text: {"rank": rank, "tasks": [], "failed": [], "nm": None, "stats": {}, "error": text}, timing)
    if timing and stats is not None:         # rank 0
        gathered = merged["gathered"]
        stats.update({k: v for k, v in gathered[0]["stats"].items() if k not in ("tasks", "weight", "inflated_bytes")})
        stats["vcf_write_s"] += merged["vcf_s"]
        stats["snf_write_s"] = merged["snf_s"]
        stats["ranks"] = [dict(p["stats"], failed=p["failed"]) for p in gathered]
        stats.update(timing)
    return written
