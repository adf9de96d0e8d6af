"""Host-side mirror of the reference's Task interface for the hot path (parallel.py:42-297):
same method names and meaning — build_leadtab / call_candidates / finalize_candidates /
execute — with the three hot calls forwarded to libsnfb200 through ctypes.

A `Task` works on one contig (one snfb_task); several tasks can share one record block and one
device run, which is how the contigs of a genome are processed per GPU.  Every device pass -- a
pass of call.call_sample or genotype.genotype_vcf, a task's own BAM region, a block handed to
`run_block` -- is packed by `pass_block` (when it comes from a BAM) and loaded and run by
`load_and_run`."""
import logging
import time
from dataclasses import dataclass, field
from typing import NamedTuple, Optional

import numpy as np

from . import abi, binding, postprocess

_CTX = {}      # per-process device contexts, created lazily after fork; never pickled (SURVEY 8b)


def device_context(device: int = 0) -> binding.Context:
    if device not in _CTX:
        _CTX[device] = binding.Context(device)
    return _CTX[device]


_REF = {}      # per device context: ((FASTA path, loaded contigs), the fasta.Reference resident on it, or None when it could not be loaded)


def reference_for(ctx, path, contigs=None):
    """the reference FASTA resident on `ctx`, loaded on first use.  contigs: the names to load (None: all), as one rank of a multi-GPU
    run loads only the contigs of its tasks; every caller of a run passes the same names, so the N mask and the VCF writer share one
    object.  A context holds one genome: another path or set of names is loaded in place of the last one, whose object is dropped (its
    gathers would read the new genome).  A FASTA that cannot be opened or read (a missing or stale index, a damaged BGZF block) is logged
    once as the reference logs it (vcf.py:116-119) and the run goes on without it."""
    key = (str(path), None if contigs is None else tuple(sorted(set(contigs))))
    held = _REF.get(ctx)
    if held is None or held[0] != key:
        from . import fasta
        try:
            ref = fasta.Reference(path, ctx, contigs=contigs)
        except (OSError, ValueError, RuntimeError) as e:
            logging.error(f"Unable to open reference file {path}: {e}")
            ref = None
        _REF[ctx] = held = (key, ref)
    return held[1]


def mask_block(block, config, ctx, regions=None, contigs=None):
    """with config.reference: the block's N-mask tables from the reference loaded on `ctx` (LeadProvider._mask_N_coverage,
    leadprov.py:420-443), before the block is loaded; without it the block is left as it is.  regions: {task index: [(start, end)]};
    contigs: the names reference_for loads (None: all)"""
    if getattr(config, "reference", None):
        ref = reference_for(ctx, config.reference, contigs)
        if ref is not None:
            from . import fasta
            fasta.mask_block(block, ref, regions)
    return block


def fetch_windows(contig, start, end, regions):
    """the (start, end) of every bam.fetch a task makes, in order: its regions [(contig, start, end)] as given (LeadProvider.build_leadtab, leadprov.py:445-470),
    else its own [start, end) (parallel.py:101).  A window pysam's parse_region refuses raises its ValueError (restated, not pinned: start <
    0, or start > end), which fails the task in the reference's worker."""
    windows = [(int(r[1]), int(r[2])) for r in regions] if regions else [(int(start), int(end))]
    for s, e in windows:
        if s < 0:
            raise ValueError(f"start out of range ({s})")
        if s > e:
            raise ValueError(f"invalid coordinates: start ({s}) > stop ({e})")
    return windows


def region_table(windows_by_task):
    """abi.REGION_DTYPE rows of [(task index, [(start, end), ...])] in task order, or None when no task has regions"""
    rows = [(t, s, e, 0) for t, w in windows_by_task for s, e in w]
    return np.array(rows, dtype=abi.REGION_DTYPE) if windows_by_task else None


@dataclass
class BlockRun:
    """Result of the device pass over one record block, shared by the tasks of that block."""
    block: object
    result: object
    cand_range: list          # per task (lo, hi) into result.cand
    rec_nm: Optional[np.ndarray] = None
    genotype: Optional[dict] = None   # per task index: snfb_genotype_targets results of the task's targets (genotype.device_targets)
    read_names: Optional[binding.ReadNames] = None    # with --output-rnames: the candidates' read names (read_names)


def read_names(ctx):
    """the read names of the run resident on `ctx` (snfb_read_names), a warning logged when two reads of a candidate share a 64-bit name hash"""
    names = ctx.read_names()
    if names.collisions:
        logging.warning(f"{names.collisions} supporting read(s) share a 64-bit read name hash with another read of their SV candidate: "
                        "RNAMES lists one name per hash")
    return names


class TaskInput(NamedTuple):
    """one task of a device pass (call.task_inputs): bamio.BamFile.device_input over its fetch windows (BGZF bytes and spans), the bytes
    snfb_load_bam inflates them to, and its fetch windows when its contig has regions (else None)"""
    id: int
    contig: str
    start: int
    end: int
    bgzf: Optional[np.ndarray]
    spans: Optional[np.ndarray]
    inflated: Optional[int]
    regions: Optional[list]


def pass_block(ctx, bam, items, config, tandem_repeats, contigs=None, records=()):
    """the record block of one device pass over `items` (TaskInput; the k-th is task index k of the block): the task, contig and
    tandem-repeat tables of bamio.pack_records, then mask_block with the tasks' regions.  tandem_repeats: {contig: intervals}
    (load_tandem_repeats); contigs: the names reference_for loads (None: all); records: host-decoded (task index, record, region index)
    packed with the tables (the host reader; snfb_load_bam needs none)."""
    from . import bamio
    tr = {k: [(int(a), int(b)) for a, b in tandem_repeats[it.contig]] for k, it in enumerate(items) if tandem_repeats.get(it.contig)}
    # a task with regions: its records carry their region's window, its own bounds only clip the N mask (the host clips it to the regions)
    bounds = [(0, bam.get_reference_length(it.contig)) if it.regions else (int(it.start), int(it.end)) for it in items]
    block = bamio.pack_records(bam.contigs, list(records), [(bam.name_to_id[it.contig], s, e, int(it.id)) for it, (s, e) in zip(items, bounds)],
                               tandem_repeats=tr or None)
    regions = {k: it.regions for k, it in enumerate(items) if it.regions}
    # mask_block's optional arguments go only to a pass that uses them: without regions or a contig subset the call stays
    # mask_block(block, config, ctx), the form a stand-in N mask (tests/test_gpu_reference.py) replaces
    if regions or contigs is not None:
        return mask_block(block, config, ctx, regions or None, contigs)
    return mask_block(block, config, ctx)


def load_and_run(ctx, config, block, windows=None, bgzf=None, spans=None, cigar16=True):
    """one device pass over `block` on `ctx`: set_config, set_regions (windows: [(task index, [(start, end)])] of every task when some task
    has regions, else None), the load -- snfb_load_bam of `bgzf` / `spans` into the block's tables, or without them snfb_load_records of
    the block's own records (cigar16 as Context.load takes it) -- and snfb_run; with config.output_rnames also the candidates' read names
    (read_names), before the next load replaces the records.  Returns the BlockRun and its split {"load_bam_s", "run_s"}, with the read
    names also "rnames_s"."""
    ctx.set_config(abi.Config.from_sniffles(config))
    t0 = time.perf_counter()
    ctx.set_regions(region_table(windows) if windows else None)
    if bgzf is not None:
        n_rec = ctx.load_bam(bgzf, spans, block)["n_rec"]
    else:
        ctx.load(block, cigar16=cigar16)
        n_rec = len(block.rec)
    t1 = time.perf_counter()
    res = ctx.run(want_leads=True, want_cands=True, want_seqs=True)
    t2 = time.perf_counter()
    split = {"load_bam_s": t1 - t0, "run_s": t2 - t1}
    names = None
    if getattr(config, "output_rnames", False):
        names = read_names(ctx)
        split["rnames_s"] = time.perf_counter() - t2
    rec_nm = abi.view(res._rec_nm_ptr, "<f8", n_rec).copy() if getattr(res, "_rec_nm_ptr", None) else None
    return BlockRun(block, res, cand_ranges(res.cand, len(block.task)), rec_nm, read_names=names), split


def run_block(block, config, device: int = 0, ctx=None) -> BlockRun:
    """leadprov -> cluster -> consensus for every task of an already packed block in one device pass (no N mask: the caller masks the
    block)."""
    return load_and_run(ctx or device_context(device), config, block)[0]


def cand_ranges(cand, n_task):
    t = cand["task"]
    lo = np.searchsorted(t, np.arange(n_task), side="left")
    hi = np.searchsorted(t, np.arange(n_task), side="right")
    return list(zip(lo.tolist(), hi.tolist()))


_BAM = {}      # per-process open BAM files (path -> bamio.BamFile)


def open_bam(path):
    from . import bamio
    if path not in _BAM:
        _BAM[path] = bamio.BamFile(path)
    return _BAM[path]


def gpu_count():
    """GPUs this process may use: SNFB_N_GPUS, else what the CUDA runtime reports (the worker with id w binds to w % n, SURVEY 8b)"""
    import os
    if os.environ.get("SNFB_N_GPUS"):
        return max(1, int(os.environ["SNFB_N_GPUS"]))
    try:
        import torch
        return max(1, torch.cuda.device_count())
    except Exception:
        return 1


def load_tandem_repeats(filename, padding):
    """util.load_tandem_repeats (util.py:121-147): BED of tandem repeats -> {contig: [(start - padding clipped at 0, end + padding), ...]},
    in file order unless some contig's starts go backwards, in which case every contig is sorted (the reference sorts all of them then).
    The result is what `Task(tandem_repeats=...)` takes per contig (sniffles:313-358)."""
    contigs_tr, unsorted = {}, False
    with open(filename, "r") as handle:
        for line in handle:
            parts = line.split("\t")
            if len(parts) >= 3:
                contig, start, end = parts[0], int(parts[1]), int(parts[2])
                iv = contigs_tr.setdefault(contig, [])
                if iv and start < iv[-1][0]:              # compared with the previous PADDED start, as the reference does (util.py:134-136)
                    unsorted = True
                iv.append((max(0, start - padding), end + padding))
    if unsorted:
        for contig in contigs_tr:
            contigs_tr[contig].sort()
    return contigs_tr


def should_process_contig(contig, length, config):
    """util.should_process_contig (util.py:150-164): --contig, --regions and, without --all-contigs, the 1 Mb rule"""
    regions = getattr(config, "regions_by_contig", None) or {}
    if config.contig and contig not in config.contig:
        return False
    if regions and contig not in regions:
        return False
    if not config.all_contigs and length < 1_000_000:
        return bool((config.contig and contig in config.contig) or (contig in regions))
    return True


def plan(contigs, config):
    """the task plan of a BAM header for call_sample and genotype_vcf (sniffles:311-358 with task_count_multiplier 0): contigs = [(name,
    length)] in header order.  Returns (processed, planned): processed = [(name, length)] of every contig should_process_contig keeps (the
    VCF header's contigs and the SNF's contig list); planned = [(task id, name, 0, length - 1)], one task per processed contig longer than
    one base, task ids counted over the planned tasks only, as the reference numbers them."""
    processed, planned = [], []
    for name, length in contigs:
        if not should_process_contig(name, length, config):
            continue
        processed.append((name, length))
        if length - 1 > 0:
            planned.append((len(planned), name, 0, length - 1))
    return processed, planned


@dataclass
class Task:
    id: int
    sv_id: int
    contig: str
    start: int
    end: int
    config: object
    assigned_process_id: Optional[int] = None
    lead_provider: object = None
    bam: object = None
    tandem_repeats: list = None
    genotype_svs: list = None
    regions: list = None
    result: object = None
    # the device pass this task reads from, and its index in that block.  Either handed in (several tasks sharing one block and one
    # device pass: call.load_pass, run_block), or built by the task itself from its BAM region on first use, the way the reference's
    # worker does.
    block_run: BlockRun = None
    task_index: int = 0
    coverage_average_total: float = 0.0
    device: int = 0
    device_ingest: bool = True      # a task that reads its own BAM region ships the COMPRESSED bytes: inflate + record decode on the GPU (snfb_load_bam)

    # ---- the reference's way: Task(id, sv_id, contig, start, end, config, bam=..., tandem_repeats=...) and a worker (parallel.py:47-60, 741-746)
    def _open(self):
        bam = self.bam if self.bam is not None else getattr(self.config, "input", None)
        if isinstance(bam, str):
            bam = open_bam(bam)
        if bam is None:
            raise RuntimeError("Task has neither a block_run nor a BAM to read its region from")
        return bam

    def _ctx(self):
        return device_context(self.device)

    def label(self):
        return f"{type(self).__name__}(id={self.id}, contig={self.contig}, start={self.start}, end={self.end})"

    def log_failure(self, log, err, failed=None):
        """the reference worker's error line for this task, which fails and is left out; failed: receives (task id, contig, error class
        name)"""
        log.error(f"Error in worker process while executing {self.label()}: {err}")
        if failed is not None:
            failed.append((self.id, self.contig, type(err).__name__))

    def bind(self, worker=None):
        """device = worker.id % n_gpus: a context per process and device, created lazily after the fork"""
        if worker is not None and getattr(worker, "id", None) is not None:
            self.device = int(worker.id) % gpu_count()
        return self

    def build_leadtab(self):
        """parallel.py:90-102 — returns (externals, read_count).  Leads outside the region are dropped on the
        device, exactly as the caller discards `externals` (parallel.py:264).  Without a block_run the task first runs its own BAM
        region (`self.bam`: an open bamio.BamFile or a path; default config.input) as a one-task device pass."""
        if self.block_run is None:
            ctx = self._ctx()
            windows = fetch_windows(self.contig, self.start, self.end, self.regions)
            bam = self._open()
            if self.device_ingest:
                # the reference's `bam.fetch(contig, start, end)` (parallel.py:95-98, leadprov.py:488) with htslib's work on the GPU: the host
                # only resolves the BAI index; BGZF inflate, record decode, region filter and CIGAR16 packing are snfb_load_bam
                bgzf, spans = bam.device_input([(self.contig, s, e) for s, e in windows], tags=[(0, g) for g in range(len(windows))])
                recs = ()
            else:
                # the host reader (also what the tests compare the device ingest with): records decoded and packed region by region
                bgzf = spans = None
                recs = [(0, r, g) for g, (s, e) in enumerate(windows) for r in bam.fetch(self.contig, s, e)]
            regions = windows if self.regions else None
            item = TaskInput(self.id, self.contig, self.start, self.end, bgzf, spans, None, regions)
            block = pass_block(ctx, bam, [item], self.config, {self.contig: self.tandem_repeats}, records=recs)
            # the host reader ships BAM CIGAR words: the library converts them (snfb_load_records)
            self.block_run, _ = load_and_run(ctx, self.config, block, [(0, windows)] if regions else None, bgzf, spans, cigar16=False)
            self.task_index = 0
        r = self.block_run.result
        self.config.average_regional_nm = float(r.task_mean_nm[self.task_index])      # leadprov.py:577-578
        self.config.qc_nm_threshold = self.config.average_regional_nm
        return [], int(r.task_read_count[self.task_index])

    def call_candidates(self, keep_qc_fails, config):
        """parallel.py:104-127"""
        br = self.block_run
        lo, hi = br.cand_range[self.task_index]
        need_leads = bool(config.mosaic) or bool(config.phase)
        calls = postprocess.calls_from_result(br.result, self.task_index, lo, hi, br.block.contig_names, self.contig, self.id, config,
                                              rec_nm=br.rec_nm, want_leads=need_leads,
                                              names=br.read_names if getattr(config, "output_rnames", False) else None)
        self.sv_id += len(calls)
        self.coverage_average_total = float(br.result.task_cov_mean[self.task_index])
        return calls

    def finalize_candidates(self, candidates, keep_qc_fails, config):
        """parallel.py:129-201"""
        return postprocess.finalize_candidates(candidates, keep_qc_fails, config, self.coverage_average_total)


def first_unanchored_bnd(calls):
    """the first BND candidate of a task with no non-BND candidate before it, or None.  postprocessing.coverage (postprocessing.py:81-90)
    leaves `end` unbound for such a BND and raises UnboundLocalError, which fails the whole task in the reference's worker."""
    return calls[0] if calls and calls[0].svtype == "BND" else None


class CallTaskError(RuntimeError):
    """the task fails as the reference's worker fails it (parallel.py:747-752): none of its records or SNF candidates are written"""


class CallTask(Task):
    # with config.snf, the task's SNF part after execute: (task id, contig, block index {block: (offset, length)}, part bytes, candidate
    # count, coverage_average_total) -- what CallResult carries to SNFile.write_results (parallel.py:279-294); snf.write_results joins them
    snf_part: Optional[tuple] = None

    def execute(self, worker=None):
        """parallel.py:256-297.  Returns (calls, read_count): the calls the VCF gets, QC fails dropped unless --no-qc, sorted by position
        with config.sort.  With config.snf the task also builds its SNF part in memory (`snf_part`), as the reference writes its
        temporary part file: every candidate after finalize, QC fails included, stored by SNFWriter, each block's `_COVERAGE` from
        snfb_coverage_bins over the block loaded on the task's device context, then write_and_index."""
        config = self.config
        self.bind(worker)
        qc = not (config.snf is not None or config.no_qc)
        _, read_count = self.build_leadtab()
        cands = self.call_candidates(qc, config)
        bad = first_unanchored_bnd(cands)
        if bad is not None:
            raise CallTaskError(f"candidate {bad.id} is a BND with no earlier non-BND candidate in its task")
        calls = self.finalize_candidates(cands, not qc, config)
        if config.snf is not None:
            import io
            from . import snf
            buf = io.BytesIO()
            part = snf.SNFWriter(config, buf)
            for c in calls:
                part.store(c)
            part.annotate_block_coverages(self._ctx().coverage_bins(self.task_index, config.coverage_binsize_combine))
            part.write_and_index()
            self.snf_part = (self.id, self.contig, dict(part.index), buf.getvalue(), len(calls), self.coverage_average_total)
        if not config.no_qc:
            calls = [c for c in calls if c.qc]
        if config.sort:
            calls = sorted(calls, key=lambda c: c.pos)
        self.result = calls
        return calls, read_count


class GenotypeTaskError(RuntimeError):
    """the task fails as the reference's worker fails it: its targets are not written"""


class GenotypeTask(Task):
    def execute(self, worker=None):
        """parallel.py:300-369: candidates finalized with QC fails kept, each target matched to the nearest candidate of its bins and
        probed for coverage on the device (snfb_genotype_targets), then genotyped.  Returns (targets, read_count)."""
        from . import genotype
        config = self.config
        self.bind(worker)
        _, read_count = self.build_leadtab()
        cands = self.call_candidates(False, config)
        calls = self.finalize_candidates(cands, True, config)
        targets = list(self.genotype_svs or [])
        bad = first_unanchored_bnd(calls)   # postprocessing.coverage over the candidates raises UnboundLocalError before any target is looked at
        if bad is not None:
            raise GenotypeTaskError(f"candidate {bad.id} is a BND with no earlier non-BND candidate in its task")
        for t in targets:
            if t.svtype not in genotype.SVTYPE_CODE:
                genotype.log.warning(f"Unsupported SVTYPE: {t.svtype}")
        br = self.block_run
        if br.genotype is not None and self.task_index in br.genotype:
            res = br.genotype[self.task_index]
        else:
            res = genotype.device_targets(self._ctx(), [(self.task_index, targets)], {n: i for i, n in enumerate(br.block.contig_names)}, config)[self.task_index]
        match, cov_start, cov_center, cov_end, bnd_no_prev = res
        if bnd_no_prev.any():
            # postprocessing.coverage raises UnboundLocalError for a BND with no earlier non-BND target in the task (postprocessing.py:81-90)
            raise GenotypeTaskError(f"BND target at line {targets[int(np.argmax(bnd_no_prev))].raw_vcf_line_index} has no earlier non-BND target in its task")
        by_index = {c.cand_index: c for c in calls}
        for t, m, s, c, e in zip(targets, match.tolist(), cov_start.tolist(), cov_center.tolist(), cov_end.tolist()):
            t.genotype_match_sv = by_index[m] if m >= 0 else None
            t.coverage_start, t.coverage_center, t.coverage_end = s, c, e
        self.result = targets
        return targets, read_count
