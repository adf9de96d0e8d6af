"""Combining samples from the command line (`sniffles -i a.snf b.snf ... -v out.vcf`, or `-i samples.tsv`): the combine run mode of
sniffles:371-481, parallel.py:372-572 and result.py:133-243.

  * the sample list comes from the SNF paths or a .tsv, each SNF header is read and checked, and the contigs are the last header's
    config.contig_lengths, filtered by --contig / --regions;
  * one combine.CombineTask per contig over its blocks (or the blocks its regions touch), split by `scatter` as the reference splits it;
  * tasks run in passes of consecutive tasks whose candidate count fits a budget: the host unpickles a pass's SNF blocks into flat columns
    (FlatPass), one snfb_combine_plan call plans the chunks and groups them on the device, and combine.CombineTask.emit_batches calls the
    groups on the host;
  * with --combine-population, the population SNF's variants of the planned contigs are loaded to the device once, and every call a pass
    makes gets POPULATION_AF / POPULATION_SIZE from one snfb_population_match call (SVGroup.call, sv.py:475-479);
  * each task's calls are ordered as CombineResult orders them, or, above --combine-max-inmemory-results inputs, as CombineResultTmpFile
    keeps them (a sorted batch's calls below the task's highest stored position are dropped), and written through vcf.open_output;
  * with --reference, the FASTA's planned contigs are loaded to the device once (tasks.reference_for, as sniffles:253-256 and
    result.py:210-214 open it for the writer of either ordering), every allele interval the records of a pass can ask for is gathered in
    one Reference.prefetch, and VCFWriter.write_call takes REF / ALT from it after the population annotation;
  * with --gpus N > 1, under torchrun, every rank plans alike, runs the tasks dist.lpt_assign gives it over their SNF bytes
    (dist.combine_task_weights) and formats their records into text, and rank 0 writes the file of one GPU (combine_snfs_ranks).

Deviations from the reference: an SNF that is missing, unreadable or whose header has no contig_lengths is refused with a message instead
of a traceback; a header without snf_format_version (as this package's SNF writer leaves it) is taken as the current version; the dropped
calls of CombineResultTmpFile are counted and logged, not written to an `-unsorted.part.vcf`; a population SNF that is missing, has no
`population` header record or holds blocks that are not PopulationVariant lists is refused before any output is opened; an INS population
variant with svlen 0 that reaches the alignment test, where the reference's worker divides by zero, stops the run with a message naming
it; a FASTA that cannot be opened is logged once, where CombineResultTmpFile logs it for every task's part (on several GPUs, once by
every rank that cannot read its contigs of it, and every rank then runs without it, as one GPU does).  On several GPUs a run in which any rank fails writes no file at all, and every rank raises the same CombineError
naming the first failed rank and its message, where one GPU leaves a plain .vcf written up to the failure."""
import contextlib
import logging
import os
import time

import numpy as np

from . import call, combine, postprocess, snf, tasks, vcf
from .snf import TYPES

log = logging.getLogger("sniffles_b200.combine")

SNF_FORMAT_VERSION = "S2_rc4"             # config.py:31
REQC_BUILD = "2.5.3"                      # snf.py:78: files of older builds are re-QC'd with --re-qc auto
TARGET_WORK_PER_TASK = 10000              # parallel.CombineTask.TARGET_WORK_PER_TASK
# Candidates one pass may hold.  Host memory is the bound: an unpickled candidate takes about 1 KB of Python objects, the device about 20
# bytes per sample plus 200 bytes.
PASS_CANDIDATES = 2_000_000


class CombineError(RuntimeError):
    """the run stops as the reference's util.fatal_error_main stops it; the message is the reference's where it has one"""


def parse_reqc(value):
    """--re-qc: 'auto', or 0 / 1 (config.py:526-531)"""
    if value == "auto":
        return "auto"
    if value in ("0", "1"):
        return bool(int(value))
    raise CombineError("Invalid value for --re-qc, allowed values are: auto, 0, 1")


def needs_reqc(header, reqc):
    """SNFile.reqc (snf.py:66-81): with 'auto', a file without config.build, or whose build before the first '-' compares below '2.5.3'
    as a string, is re-QC'd"""
    if reqc != "auto":
        return reqc
    try:
        build, _, _ = header["config"]["build"].partition("-")
    except (KeyError, AttributeError, TypeError):
        return True
    return build < REQC_BUILD


def sample_list(inputs):
    """[(SNF path, sample id or None)] of the inputs (sniffles:380-407): a single .tsv lists one SNF per line, optionally with a sample
    id in a second tab-separated column; blank lines and lines starting with '#' are skipped"""
    if len(inputs) == 1 and inputs[0].split(".")[-1].lower() == "tsv":
        out = []
        try:
            with open(inputs[0], "r") as f:
                lines = f.readlines()
        except OSError as e:
            raise CombineError(f"Unable to read the sample list {inputs[0]}: {e}") from e
        for i, line in enumerate(lines):
            s = line.strip()
            if len(s) == 0 or s[0] == "#":
                continue
            parts = s.split("\t")
            if len(parts) not in (1, 2):
                raise CombineError(f"Invalid sample list .tsv : {inputs[0]} : Line {i + 1} - expected either one or two columns (first column: "
                                   f".snf filename, second column: optional sample id to overrule the one specified in the .snf file)")
            out.append((parts[0], parts[1] if len(parts) == 2 else None))
        return out
    if inputs[0].split(".")[-1].lower() == "snf":
        return [(p, None) for p in inputs]
    raise CombineError("Failed to determine .snf files to be combined. Please specify either one or more .snf files OR a single .tsv file "
                       "as input for multi-calling.")


def read_header(path):
    try:
        r = snf.SNFReader(path)
    except (OSError, ValueError, KeyError, UnicodeDecodeError) as e:
        raise CombineError(f"Unable to read the SNF file {path}: {e}") from e
    r.close()
    return r.header


def _contig_lengths(header, path):
    cl = header.get("config", {}).get("contig_lengths")
    try:
        out = [(str(name), int(length)) for name, length in cl]
    except (TypeError, ValueError):
        raise CombineError(f"The header of {path} has no contig_lengths: it cannot be combined") from None
    return out


def read_inputs(config):
    """the header pass of sniffles:371-437 -> (contig lengths to process, {internal id: re-QC}).  Sets config.snf_input_info and
    config.sample_ids_vcf."""
    reqc = parse_reqc(config.re_qc)
    config.snf_input_info, config.sample_ids_vcf = [], []
    requalify, contig_lengths = {}, []
    for internal_id, (path, sample_id) in enumerate(sample_list(config.input)):
        header = read_header(path)
        hc = header.get("config", {})
        if not config.dev_skip_snf_validation:
            if hc.get("snf_block_size") != config.snf_block_size:
                raise CombineError(f"SNF block size differs for {path}")
            if hc.get("snf_format_version", SNF_FORMAT_VERSION) != SNF_FORMAT_VERSION:
                raise CombineError(f"SNF format version for {path} is not supported")
        if sample_id is None:
            sample_id = hc.get("sample_id") if hc.get("sample_id") is not None else os.path.splitext(os.path.basename(path))[0]
        contig_lengths = _contig_lengths(header, path)
        requalify[internal_id] = needs_reqc(header, reqc)
        config.snf_input_info.append({"internal_id": internal_id, "sample_id": sample_id, "filename": path})
        config.sample_ids_vcf.append((internal_id, sample_id))
        log.info(f"    {path} (sample ID in output VCF='{sample_id}'{' (Rerunning QC)' if requalify[internal_id] else ''})")
    to_process = config.contig or config.regions_by_contig
    if to_process:
        contig_lengths = [(name, length) for name, length in contig_lengths if name in to_process]
    return contig_lengths, requalify


def block_indices(start, end, regions, block_size):
    """CombineTask.generate_blocks (parallel.py:388-402): the blocks of [start, end], or the sorted union of the blocks each region touches"""
    if regions:
        out = set()
        for _, rs, re_ in regions:
            out |= set(range(rs // block_size * block_size, re_ + block_size, block_size))
        return sorted(out)
    return list(range(start, end + block_size, block_size))


def scatter(task, n_samples, threads):
    """CombineTask.scatter (parallel.py:420-441): with more than TARGET_WORK_PER_TASK blocks x samples and --threads > 1, the task becomes
    clones of total // TARGET_WORK_PER_TASK consecutive blocks each, the i-th with id task.id + i + 1"""
    total = len(task.block_indices) * n_samples
    if total <= TARGET_WORK_PER_TASK or threads <= 1:
        return [task]
    per = total // TARGET_WORK_PER_TASK
    bs = task.config.snf_block_size
    out = []
    for i, fb in enumerate(range(0, len(task.block_indices), per)):
        blocks = task.block_indices[fb:fb + per]
        out.append(combine.CombineTask(task.id + i + 1, task.contig, blocks[0], blocks[-1] + bs, task.config, block_indices=blocks))
    return out


def plan_tasks(config, contig_lengths):
    """one CombineTask per contig, scattered; the next contig's id follows the last clone's (sniffles:466-481)"""
    out, tid = [], 0
    for name, length in contig_lengths:
        regions = config.regions_by_contig.get(name)
        t = combine.CombineTask(tid, name, 0, length - 1, config, block_indices=block_indices(0, length - 1, regions, config.snf_block_size))
        out.extend(scatter(t, len(config.sample_ids_vcf), config.threads))
        tid = out[-1].id + 1
    return out


def stored_calls(pairs, tmpfile, sort):
    """[(batch, call)] of one task in emission order -> (the calls its result writes, in order, and the number dropped).  CombineResult
    (tmpfile False) sorts the task's calls by pos when sorting is on; CombineResultTmpFile sorts each batch and drops the calls of a batch
    whose pos is below the highest pos stored before it (result.py:176-206)"""
    if not tmpfile:
        calls = [c for _, c in pairs]
        return (sorted(calls, key=lambda c: c.pos) if sort else calls), 0
    out, dropped, highest, k = [], 0, -1, 0
    while k < len(pairs):
        j = k
        while j < len(pairs) and pairs[j][0] == pairs[k][0]:
            j += 1
        batch = [c for _, c in pairs[k:j]]
        k = j
        if sort:
            batch.sort(key=lambda c: c.pos)
            m = 0
            while m < len(batch) and batch[m].pos < highest:
                m += 1
            dropped += m
            highest = batch[-1].pos
            batch = batch[m:]
        out.extend(batch)
    return out, dropped


def requalify(cand, config):
    """postprocessing.genotype_sv(cand, config) as the reference runs it on a re-QC'd file's candidate: the phase is the one its
    genotype already carries"""
    gt = cand.genotypes.get(0) if isinstance(cand.genotypes, dict) else None
    phase = gt[5] if gt is not None and len(gt) > 5 else None
    postprocess.genotype_sv(cand, config, phase)


class FlatPass:
    """The SNF candidates of consecutive tasks as the flat columns snfb_combine_plan reads, in the reference's iteration order (task,
    block, svtype, sample, part, list position).  A coverage row is made for each (task, block) where some sample has the block, from the
    first part of each sample's block (parallel.py:544-545)."""

    def __init__(self, config):
        self.config = config
        self.ids = [s["internal_id"] for s in config.snf_input_info]
        self.cands, self.tasks, self.row_bpos = [], [], []
        self.cols = {k: [] for k in ("task", "row", "svtype", "support", "pos", "svlen", "sample", "mate_contig", "mate_pos")}
        self.alts, self.cov_rows, self.block_start, self.contig_ids = [], [], [], {}

    def add_task(self, task, readers):
        """decodes one task's blocks"""
        k = len(self.tasks)
        self.tasks.append(task)
        c = self.cols
        for bpos, block_index in enumerate(task.block_indices):
            sblocks = [readers[sid].read_blocks(task.contig, block_index) for sid in self.ids]
            if all(b is None for b in sblocks):
                continue
            row = len(self.cov_rows)
            self.cov_rows.append(combine.coverage_rows(sblocks, block_index, self.config))
            self.block_start.append(block_index)
            self.row_bpos.append(bpos)
            for ti, t in enumerate(combine.TYPES):
                for si, parts in enumerate(sblocks):
                    if parts is None:
                        continue
                    for blk in parts:
                        for cand in blk[t]:
                            cand.sample_internal_id = self.ids[si]
                            cand._sample_index = si
                            self.cands.append(cand)
                            c["task"].append(k)
                            c["row"].append(row)
                            c["svtype"].append(ti)
                            c["support"].append(cand.support)
                            c["pos"].append(cand.pos)
                            c["svlen"].append(cand.svlen)
                            c["sample"].append(si)
                            if t == "BND":
                                c["mate_contig"].append(self.contig_ids.setdefault(cand.bnd_info.mate_contig, len(self.contig_ids)))
                                c["mate_pos"].append(cand.bnd_info.mate_ref_start)
                            else:
                                c["mate_contig"].append(0)
                                c["mate_pos"].append(0)
                            a = cand.alt
                            self.alts.append(a.encode("latin-1") if isinstance(a, str) else bytes(a or b""))

    def arrays(self):
        """the numpy columns (binding.Context.combine_plan)"""
        cfg = self.config
        step = cfg.coverage_binsize_combine
        per_block = cfg.snf_block_size // step
        d = {k: np.asarray(v, dtype="<u4" if k in ("task", "row", "sample") else "<i4") for k, v in self.cols.items()}
        d["alt_len"] = np.fromiter((len(x) for x in self.alts), "<u4", len(self.alts))
        d["alt_off"] = np.zeros(len(self.alts), "<u8")
        if self.alts:
            d["alt_off"][1:] = np.cumsum(d["alt_len"][:-1], dtype=np.uint64)
        d["alt"] = np.frombuffer(b"".join(self.alts) + b"\0", np.uint8).copy()
        d["cov"] = np.ascontiguousarray(np.stack(self.cov_rows).astype(np.int32) if self.cov_rows else np.zeros((0, len(self.ids), per_block), np.int32))
        d["block_start"] = np.array(self.block_start, np.int64)
        d.update(bins_per_block=per_block, cov_binsize=step, n_samples=len(self.ids), n_task=max(1, len(self.tasks)))
        return d

    def plan(self, res, flat):
        """the device result of snfb_combine_plan as a combine.Plan (candidates in slot order, chains and chunks as CombineTask.plan
        builds them) and the `out` tuple CombineTask.emit reads"""
        perm = res["perm"]
        p = combine.Plan()
        p.cands = [self.cands[i] for i in perm.tolist()]
        for c0, nc, k0, nk, _, _ in res["chains"].tolist():
            f = int(perm[c0])
            p.chains.append((int(flat["task"][f]), int(flat["svtype"][f]), c0, nc, k0, nk))
        p.chunks = [(c0, nc, b, size, row, self.row_bpos[row]) for c0, nc, b, size, row, _ in res["chunks"].tolist()]
        p.cov_blocks, p.cov_rows = self.block_start, self.cov_rows
        return p, (res["cand_group"], res["emit_chunk"], res["emit_ord"], res["cov_non"])


def join(parts):
    """one FlatPass of several, in order: task indices, coverage rows and BND mate contig numbers renumbered"""
    out = FlatPass(parts[0].config)
    for b in parts:
        nt, nr = len(out.tasks), len(out.cov_rows)
        remap = {i: out.contig_ids.setdefault(name, len(out.contig_ids)) for name, i in b.contig_ids.items()}
        out.tasks += b.tasks
        out.cands += b.cands
        out.row_bpos += b.row_bpos
        out.cov_rows += b.cov_rows
        out.block_start += b.block_start
        out.alts += b.alts
        c = out.cols
        c["task"] += [v + nt for v in b.cols["task"]]
        c["row"] += [v + nr for v in b.cols["row"]]
        c["mate_contig"] += [remap[v] if t == 4 else v for v, t in zip(b.cols["mate_contig"], b.cols["svtype"])]
        for key in ("svtype", "support", "pos", "svlen", "sample", "mate_pos"):
            c[key] += b.cols[key]
    return out


def check_outputs(config):
    """the reference's checks before it reads any SNF (sniffles:122-127, 238-248): --snf is refused in this mode, --vcf is needed"""
    if config.snf is not None:
        raise CombineError("--snf cannot be used with run mode combine")
    if config.vcf is None:
        raise CombineError("Please specify at least one of: --vcf or --snf for output (both may be used at the same time)")
    try:
        call.check_outputs(config)
    except call.CallSampleError as e:
        raise CombineError(str(e)) from None


class Population:
    """the population SNF of --combine-population: its variants in the contigs of the run, flattened in file order (contig, block in
    index order, svtype, list position), with the columns snfb_population_load reads"""

    def __init__(self, path, contigs):
        where = f"the population SNF {path} (--combine-population)"
        try:
            r = snf.PopulationReader(path)
        except (OSError, ValueError, KeyError, UnicodeDecodeError) as e:
            raise CombineError(f"Unable to read {where}: {e}") from e
        try:
            if not isinstance(r.population, dict):
                raise CombineError(f"{where} has no population record in its header: it is not a population SNF")
            self.info, self.contig_ids = r.population, {name: k for k, name in enumerate(contigs)}
            self.variants = []
            cols = {k: [] for k in ("contig", "block", "svtype", "pos", "svlen")}
            self.alts = []
            for name in contigs:
                try:
                    blocks = r.blocks(name)
                except Exception as e:               # a truncated member, a pickle of unknown classes, ...
                    raise CombineError(f"Unable to read the blocks of contig {name} in {where}: {e}") from e
                for block, blk in blocks:
                    for ti, t in enumerate(TYPES):
                        lst = blk.get(t, []) if isinstance(blk, dict) else None
                        if not isinstance(lst, list) or not all(isinstance(v, r.variant_class) for v in lst):
                            raise CombineError(f"Block {name}:{block} of {where} does not hold PopulationVariant lists: it is not a population SNF")
                        for v in lst:
                            self.variants.append(v)
                            cols["contig"].append(self.contig_ids[name])
                            cols["block"].append(block)
                            cols["svtype"].append(ti)
                            cols["pos"].append(v.pos)
                            cols["svlen"].append(v.svlen)
                            self.alts.append(alt_bytes(v.alt))
        finally:
            r.close()
        self.cols = {k: np.asarray(v, "<i4") for k, v in cols.items()}
        self.path = path

    def load(self, ctx):
        c = self.cols
        ctx.population_load(c["contig"], c["block"], c["svtype"], c["pos"], c["svlen"], self.alts)

    def annotate(self, ctx, calls, config):
        """PopulationSNF.get_population_AF for every call on the device, then POPULATION_AF = round(af, 5) and POPULATION_SIZE =
        genotyped_sample_count, or 0 / 0 without a match (sv.py:475-479)"""
        if not calls:
            return
        best = ctx.population_match([self.contig_ids.get(c.contig, -1) for c in calls], [TYPES.index(c.svtype) for c in calls],
                                    [c.pos for c in calls], [c.svlen for c in calls], [alt_bytes(c.alt) for c in calls],
                                    config.combine_match, config.combine_match_max, config.combine_pctseq, config.snf_block_size)
        for c, b in zip(calls, best.tolist()):
            if b == -2:                                  # a minimum length of 0 admits distance 0 only: the variant is at the call's position
                vid = next((v.id for v in self.variants if v.contig == c.contig and v.svtype == "INS" and v.svlen == 0 and v.pos == c.pos), "?")
                raise CombineError(f"The call {c.id} at {c.contig}:{c.pos} reaches the alignment test of population variant {vid} in {self.path}, "
                                   f"whose svlen is 0: the reference stops on this division by zero")
            set_population_info(c, self.variants[b] if b >= 0 else None)


def alt_bytes(a):
    return a.encode("latin-1") if isinstance(a, str) else bytes(a or b"")


def set_population_info(call, variant):
    """the two INFO values SVGroup.call sets (sv.py:475-479): round(af, 5) and the genotyped sample count, or the integers 0 and 0"""
    af, sz = (round(variant.af, 5), variant.genotyped_sample_count) if variant is not None else (0, 0)
    call.set_info("POPULATION_AF", af)
    call.set_info("POPULATION_SIZE", sz)


def combine_snfs(config, device=0, budget=None, stats=None):
    """the combine run mode: config.input (SNF files or one .tsv) -> config.vcf.  budget: the candidates one pass may hold (default
    PASS_CANDIDATES).  stats: a dict that receives the wall-clock split (header_s, decode_s, device_s, call_group_s, write_s, passes and
    per-pass task and candidate counts, dropped; with --combine-population population_s for the decode and load of the population SNF and
    population_match_s for its matches; with --reference reference_s for the FASTA load and, per pass, prefetch_s and prefetch_bytes of
    its allele gather).  Returns the number of VCF records written.

    With --gpus N > 1 and an initialised process group of N ranks (torchrun --nproc-per-node N -m sniffles_b200 ... --gpus N) the run goes
    through combine_snfs_ranks; without a process group it runs on one GPU, as it does with --gpus 1."""
    config.mode = "combine"
    gpus = getattr(config, "gpus", 1)
    if gpus > 1:
        world = call._world_size()
        if world == gpus:
            return combine_snfs_ranks(config, device, budget, stats)
        if world > 1:
            raise CombineError(f"--gpus {gpus} does not match the {world} ranks of the process group")
        log.warning(f"--gpus {gpus}: combine mode runs on one GPU without torchrun; to run it on {gpus} GPUs launch torchrun --standalone "
                    f"--nproc-per-node {gpus} -m sniffles_b200 ... --gpus {gpus}")
    st = stats if stats is not None else {}
    st.update(_new_stats())
    t0 = time.perf_counter()
    check_outputs(config)
    contig_lengths, reqc, planned, tmpfile = _prepare(config)
    st["header_s"] = time.perf_counter() - t0
    contigs = list(dict.fromkeys(t.contig for t in planned))
    ctx, pop, reference = _device_inputs(config, device, contigs, st)
    if budget is None:
        budget = PASS_CANDIDATES
    written, readers = 0, {}
    try:
        readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in config.snf_input_info}
        with contextlib.ExitStack() as stack:
            handle = vcf.open_output(config, ctx)
            if config.vcf_output_bgz:
                stack.enter_context(handle)               # compressed and indexed when the run ends without an error
            else:
                stack.callback(handle.close)
            writer = vcf.VCFWriter(config, handle, reference)
            writer.write_header(contig_lengths)

            def write(task, calls):
                return sum(writer.write_call(c) for c in calls)

            for group in call.group_passes(_decoded(config, planned, readers, st), budget, size=lambda fp: len(fp.cands)):
                written += _run_pass(ctx, join(group), config, reqc, write, tmpfile, st, pop, reference)
            t1 = time.perf_counter()
        st["write_s"] += time.perf_counter() - t1
    finally:
        for r in readers.values():
            r.close()
    _log_written(config, written, st["dropped"])
    st["wall_s"] = time.perf_counter() - t0
    return written


def _new_stats():
    return dict(passes=0, pass_tasks=[], pass_candidates=[], header_s=0.0, decode_s=0.0, device_s=0.0, call_group_s=0.0, write_s=0.0, dropped=0,
                population_s=0.0, population_match_s=0.0, reference_s=0.0, prefetch_s=[], prefetch_bytes=[])


def _prepare(config, warn=True):
    """the header pass and the plan every run of the inputs makes alike -> (contig lengths, {internal id: re-QC}, planned tasks, whether
    the results are kept as CombineResultTmpFile keeps them).  Above --combine-max-inmemory-results inputs a sorted .vcf.gz becomes the
    plain, unsorted file (sniffles:453-457).  warn: log the warnings of that ordering (one rank of several logs them)."""
    contig_lengths, reqc = read_inputs(config)
    planned = plan_tasks(config, contig_lengths)
    tmpfile = len(config.snf_input_info) > config.combine_max_inmemory_results
    if tmpfile:
        log.info("Using tmp file aggregation for merge.")
        if config.sort:
            if warn:
                log.warning(f"Sorting is not supported above --combine-max-inmemory-results ({config.combine_max_inmemory_results}) inputs: "
                            f"the calls of a task that come out of order are dropped")
            if config.vcf_output_bgz:
                config.vcf = config.vcf.removesuffix(".gz").removesuffix(".bgz")
                config.no_sort = True
                if warn:
                    log.warning("Result will be unsorted and uncompressed")
    log.info(f"Verified headers for {len(config.snf_input_info)} .snf files.")
    return contig_lengths, reqc, planned, tmpfile


def _device_inputs(config, device, contigs, st, load=True):
    """the device context of `device`, and, when `load`, with --combine-population the population SNF's variants of `contigs` (read before
    the context is made, so that a bad file is refused before any device work: sniffles:433-435, parallel.py:454-455) loaded on it, and
    with --reference the FASTA's `contigs` resident on it (sniffles:253-256; logged and left out when it cannot be read).  Returns (ctx,
    Population or None, fasta.Reference or None)."""
    pop = None
    if config.combine_population and load:
        tp = time.perf_counter()
        pop = Population(config.combine_population, contigs)
        st["population_s"] += time.perf_counter() - tp
    ctx = tasks.device_context(device)
    if pop is not None:
        tp = time.perf_counter()
        try:
            pop.load(ctx)
        except Exception as e:
            raise CombineError(f"Loading the population SNF {pop.path} (--combine-population) to the device failed: {e}") from e
        st["population_s"] += time.perf_counter() - tp
        log.info(f"Population SNF {pop.path}: {len(pop.variants)} variants in the run's contigs")
    reference = None
    if getattr(config, "reference", None) and load:
        log.info(f"Opening for reading: {config.reference}")
        tr = time.perf_counter()
        reference = tasks.reference_for(ctx, config.reference, contigs)
        st["reference_s"] = time.perf_counter() - tr
    return ctx, pop, reference


def _log_written(config, written, dropped):
    if dropped:
        log.warning(f"{dropped} calls came out of position order in their task and were left out (CombineResultTmpFile)")
    log.info(f"Wrote {written} called SVs to {config.vcf}")


def _decoded(config, planned, readers, st):
    for task in planned:
        t0 = time.perf_counter()
        fp = FlatPass(config)
        fp.add_task(task, readers)
        st["decode_s"] += time.perf_counter() - t0
        yield fp


def _run_pass(ctx, fp, config, reqc, write, tmpfile, st, pop=None, reference=None):
    """one device call for the pass's tasks, SVGroup.call on the host, the population annotation of every call the pass made (one device
    call), with `reference` the allele intervals of every call the pass stores (one device gather), then write(task, its stored calls) ->
    records written, per task in task order; returns the records written"""
    from . import binding
    flat = fp.arrays()
    t0 = time.perf_counter()
    try:
        res = ctx.combine_plan(flat, config)
    except binding.SnfbError as e:
        raise CombineError(f"the device pass over {len(fp.tasks)} task(s) from task {fp.tasks[0].id} ({len(fp.cands)} candidates) failed: {e}") from e
    t1 = time.perf_counter()
    plan, out = fp.plan(res, flat)
    for c in plan.cands:                                 # parallel.py:503-504: a re-QC'd file's kept candidates are genotyped again
        if reqc[c.sample_internal_id]:
            requalify(c, config)
    batches = combine.CombineTask.emit_batches(fp.tasks, plan, out)
    tp = time.perf_counter()
    if pop is not None:                                  # SVGroup.call annotates each call before any result ordering drops one
        try:
            pop.annotate(ctx, [c for k in range(len(fp.tasks)) for _, c in batches[k]], config)
        except binding.SnfbError as e:
            raise CombineError(f"the population match of the pass from task {fp.tasks[0].id} failed: {e}") from e
    t2 = time.perf_counter()
    st["population_match_s"] += t2 - tp
    stored = []
    for k in range(len(fp.tasks)):
        calls, dropped = stored_calls(batches[k], tmpfile, config.sort)
        st["dropped"] += dropped
        stored.append(calls)
    prefetch_s = 0.0
    if reference is not None:                            # after the annotation: the population match compares the SNF ALT
        tr = time.perf_counter()
        st["prefetch_bytes"].append(reference.prefetch(vcf.reference_intervals([c for calls in stored for c in calls], config)))
        prefetch_s = time.perf_counter() - tr
        st["prefetch_s"].append(prefetch_s)
    written = sum(write(task, calls) for task, calls in zip(fp.tasks, stored))
    st["passes"] += 1
    st["pass_tasks"].append(len(fp.tasks))
    st["pass_candidates"].append(len(fp.cands))
    st["device_s"] += t1 - t0
    st["call_group_s"] += tp - t1
    st["write_s"] += time.perf_counter() - t2 - prefetch_s
    return written


def run_rank_tasks(config, device, budget, rank, world, plan=None):
    """one rank's share of a multi-GPU combine run: the header pass and plan every rank makes alike (_prepare; its warnings logged by rank
    0 alone), the tasks dist.lpt_assign gives this rank over dist.combine_task_weights, then the pass loop of combine_snfs over them in
    task-id order under this rank's own candidate budget, each task's stored calls formatted here into VCF text.  With
    --combine-population / --reference only the contigs of this rank's tasks are loaded, and nothing when it has none.

    Before any pass, every rank reaches one all_gather_object of (set-up ok, FASTA read): a rank whose set-up failed raises its error,
    the others then run no task (the failed rank's payload names it); and when any rank could not read its contigs of the FASTA, every
    rank runs without it, as one GPU runs without a FASTA any of whose planned contigs it cannot read.  plan: a dict that receives the
    contig lengths (rank 0 writes the header from them).  Returns the payload rank 0 merges (write_rank_outputs): {"rank", "tasks":
    [(task id, VCF text, records)], "dropped", "stats", "error": None}."""
    import io
    import torch.distributed as tdist
    from . import dist
    st = _new_stats()
    t0 = time.perf_counter()
    out, readers, failure, reference = [], {}, None, None
    try:
        try:
            contig_lengths, reqc, planned, tmpfile = _prepare(config, warn=rank == 0)
            readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in config.snf_input_info}
            weights = dist.combine_task_weights(readers, planned)
            owner = dist.lpt_assign(weights, world)
            mine = [t for t, o in zip(planned, owner) if o == rank]
            st.update(tasks=len(mine), weight=sum(w for w, o in zip(weights, owner) if o == rank), header_s=time.perf_counter() - t0)
            ctx, pop, reference = _device_inputs(config, device, list(dict.fromkeys(t.contig for t in mine)), st, load=bool(mine))
            fasta_read = reference is not None or not (getattr(config, "reference", None) and mine)
        except Exception as e:               # after the all-gather below: a rank that raised before it would leave the others waiting
            failure, fasta_read = e, True
        verdicts = [None] * world
        tdist.all_gather_object(verdicts, (failure is None, fasta_read))
        if failure is not None:
            raise failure
        if not all(ok for ok, _ in verdicts):
            st["wall_s"] = time.perf_counter() - t0
            return {"rank": rank, "tasks": [], "dropped": 0, "stats": st, "error": None}
        if not all(read for _, read in verdicts):
            if reference is not None:
                log.warning("another rank could not read its contigs of the reference FASTA: this rank runs without it, as one GPU would")
            reference = None
        if plan is not None:
            plan["contig_lengths"] = contig_lengths

        def write(task, calls):
            buf = io.StringIO()
            writer = vcf.VCFWriter(config, buf, reference)
            n = sum(writer.write_call(c) for c in calls)
            out.append((task.id, buf.getvalue(), n))
            return n

        for group in call.group_passes(_decoded(config, mine, readers, st), PASS_CANDIDATES if budget is None else budget,
                                       size=lambda fp: len(fp.cands)):
            _run_pass(ctx, join(group), config, reqc, write, tmpfile, st, pop, reference)
    finally:
        for r in readers.values():
            r.close()
    st["wall_s"] = time.perf_counter() - t0
    return {"rank": rank, "tasks": out, "dropped": st["dropped"], "stats": st, "error": None}


def write_rank_outputs(config, contig_lengths, payloads, device=0):
    """rank 0's merge of every rank's payload (run_rank_tasks): when any rank failed, no file is written and CombineError names the first
    failed rank and its message; otherwise the VCF header, then every task's text in task-id order through vcf.open_output (a .vcf.gz
    compressed on `device` and indexed).  Logs the run's dropped calls and records.  Returns (records written, calls dropped)."""
    failed = [p for p in payloads if p["error"] is not None]
    if failed:
        raise CombineError(f"rank {failed[0]['rank']}: {failed[0]['error']}")
    done = sorted((t for p in payloads for t in p["tasks"]), key=lambda t: t[0])
    dropped = sum(p["dropped"] for p in payloads)
    written = 0
    ctx = tasks.device_context(device) if config.vcf_output_bgz else None
    with vcf.open_output(config, ctx) as handle:          # a .vcf.gz is compressed and indexed when the writing ends without an error
        vcf.VCFWriter(config, handle).write_header(contig_lengths)
        for _, text, n in done:
            handle.write(text)
            written += n
    _log_written(config, written, dropped)
    return written, dropped


def combine_snfs_ranks(config, device, budget=None, stats=None):
    """combine_snfs over the ranks of an initialised torch.distributed process group, through dist.rank_run: rank 0 checks the outputs
    (check_outputs; no other rank calls it) and broadcasts the verdict; every rank runs its own tasks (run_rank_tasks) and sends its
    payload to rank 0, an error included.  Rank 0 writes the file (write_rank_outputs): every rank returns the same count or raises the
    same CombineError.  Rank 0 holds every rank's VCF text at once, host memory in proportion to the output file.

    stats on rank 0: the keys of combine_snfs for rank 0's own work, with "dropped" summed over the ranks and "write_s" the time of rank
    0's merge and write (each rank's own formatting time is its "write_s" under "ranks"), plus "ranks" (per rank its split, task count
    and weight) and "gather_s"."""
    from . import dist
    plan, timing, merged = {}, {}, {}

    def write(gathered):
        # a rank 0 whose header pass failed has no contig lengths: write_rank_outputs names the failed rank before it needs them
        written, merged["dropped"] = write_rank_outputs(config, plan.get("contig_lengths", []), gathered, device)
        merged["gathered"] = gathered
        return written

    written = dist.rank_run(lambda: check_outputs(config), lambda rank, world: run_rank_tasks(config, device, budget, rank, world, plan),
                            write, CombineError, log, lambda rank, text: {"rank": rank, "tasks": [], "dropped": 0, "stats": {}, "error": text},
                            timing)
    if timing and stats is not None:         # rank 0
        gathered = merged["gathered"]
        stats.update({k: v for k, v in gathered[0]["stats"].items() if k not in ("tasks", "weight")})
        stats["dropped"] = merged["dropped"]
        stats["ranks"] = [p["stats"] for p in gathered]
        stats.update(timing)
    return written
