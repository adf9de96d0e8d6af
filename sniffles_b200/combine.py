"""Multi-sample combine — SURVEY.md §8(f)1 / E1: the host mirror of the reference's CombineTask
(/root/reference/src/sniffles/parallel.py:372-572) over SNF inputs.

Split of the work:
  * host (this module): read the SNF blocks of every sample, form the chunks the reference forms (bins of combine_min_size accumulated to
    bin_max_candidates, candidates of a chunk in support order — parallel.py:484-527, cluster.py:361) as flat arrays;
  * device (csrc/combine.cuh through snfb_combine_groups): the sequential greedy grouping of every (task, svtype) chain — resolve_block_groups,
    SVGroup.from_candidate / add_candidate, the coverage of the samples a group does not include, the keep / call split;
  * host: SVGroup.call per emitted group in the reference's emission order (sv.py:323-481).

`group.align_call` (sv.py:282-292, edlib's global edit distance between ALT strings) is evaluated on the device when config.combine_pctseq != 0
(the default 0.7); `--combine-pctseq 0` gives the reference's behaviour without edlib."""
import statistics
from dataclasses import dataclass, field

import numpy as np

from . import postprocess, snf

TYPES = snf.TYPES


@dataclass
class SVGroup:                                                   # what SVGroup.call reads of sv.SVGroup
    candidates: list
    included_samples: set
    coverages_nonincluded: dict


def _mean(nums):
    nums = list(nums)
    return sum(nums) / len(nums)


def _mean_or_none_round(nums):
    nums = list(nums)
    return None if not nums else round(sum(nums) / len(nums))


def _stdev(nums):
    nums = list(nums)
    return statistics.stdev(nums) if len(nums) > 1 else 0


def call_group(group: SVGroup, config, task):
    """SVGroup.call (sv.py:323-481), restated"""
    first = group.candidates[0]
    cands = group.candidates
    n_samples = len(config.snf_input_info)
    samples_count = float(n_samples)
    sample_internal_ids = set(s["internal_id"] for s in config.snf_input_info)
    total_count = len(group.included_samples)
    pass_count = sum(c.qc for c in cands)
    qc = ((pass_count > 0 and pass_count / samples_count >= config.combine_high_confidence) or
          (total_count / samples_count >= config.combine_low_confidence and total_count >= config.combine_low_confidence_abs))
    single_noqc = config.no_qc and n_samples == 1
    if not qc and not single_noqc:
        return None
    if not config.combine_output_filtered and not any(c.qc and c.filter == "PASS" for c in cands) and not single_noqc:
        return None
    rnames, genotypes = [], {}
    for c in cands:
        if c.rnames is not None:
            rnames.extend(c.rnames)
        if 0 not in c.genotypes:
            c.genotypes[0] = (".", ".", 0, 0, c.support, (None, None))
        a, b, gt_qual, dr, dv, ps = c.genotypes[0]
        if c.sample_internal_id in genotypes:                     # intra-sample merging
            ca, cb, cq, cdr, cdv, cps, cid = genotypes[c.sample_internal_id]
            new_id = cid + "," + config.id_prefix + c.id
            if ca == "." or (a != "." and (a, b) >= (ca, cb)):
                genotypes[c.sample_internal_id] = (a, b, gt_qual, dr, dv, ps, new_id)
            else:
                genotypes[c.sample_internal_id] = (ca, cb, cq, cdr, cdv, cps, new_id)
        else:
            genotypes[c.sample_internal_id] = (a, b, gt_qual, dr, dv, ps, config.id_prefix + c.id)
    for sid in sample_internal_ids:
        if sid in genotypes:
            continue
        coverage = group.coverages_nonincluded[sid]
        if coverage >= config.combine_null_min_coverage:
            genotypes[sid] = (0, 0, 0, coverage, 0, (None, None), "NULL")
        else:
            genotypes[sid] = (".", ".", 0, coverage, 0, (None, None), "NULL")
    if getattr(config, "combine_consensus", False):
        raise NotImplementedError("--combine-consensus unpacks 5-tuples from 7-tuples in the reference (sv.py:387) and cannot run there either")
    if config.combine_pair_relabel:
        max_gt = (0, 0)
        for sid in genotypes:
            a, b, q, dr, dv, ps, nid = genotypes[sid]
            if q > config.combine_pair_relabel_threshold and a != ".":
                max_gt = max(max_gt, (a, b))
        if max_gt != (0, 0):
            for sid in genotypes:
                a, b, q, dr, dv, ps, nid = genotypes[sid]
                if q < config.combine_pair_relabel_threshold and a != ".":
                    genotypes[sid] = (max_gt[0], max_gt[1], q, dr, dv, ps, nid)
    pos_med = int(int(statistics.median(c.pos for c in cands)))
    len_med = int(int(statistics.median(c.svlen for c in cands)))
    svlens = [l for c in cands for l in (c.svlens or [])] if getattr(config, "dev_emit_sv_lengths", False) else None
    alt = first.alt
    mind = abs(len(alt) - len_med)
    if first.svtype == "INS":
        end_med = pos_med
        for c in cands:
            d = abs(len(c.alt) - len_med)
            if d < mind:
                mind, alt = d, c.alt
    else:
        end_med = pos_med + abs(len_med)
    med = getattr(config, "dev_combine_medians", False)
    call = postprocess.SVCall(
        contig=first.contig, pos=pos_med if med else first.pos, id=f"{first.svtype}.{task.sv_id:X}M{task.id:X}", ref="N", alt=alt,
        qual=_mean_or_none_round(int(c.qual) for c in cands if c.qual is not None),
        filter="PASS" if n_samples != 1 else first.filter, info=dict() if n_samples != 1 else first.info,
        svtype=first.svtype, svlen=len_med if med else first.svlen, svlens=svlens, end=end_med if med else first.end,
        genotypes=genotypes, precise=sum(int(c.precise) for c in cands) / float(len(cands)) > 0.5,
        support=round(_mean(c.support for c in cands)), rnames=rnames, postprocess=None, qc=True, nm=-1,
        fwd=sum(c.fwd for c in cands), rev=sum(c.rev for c in cands),
        coverage_upstream=_mean_or_none_round(c.coverage_upstream for c in cands if c.coverage_upstream is not None),
        coverage_start=_mean_or_none_round(c.coverage_start for c in cands if c.coverage_start is not None),
        coverage_center=_mean_or_none_round(c.coverage_center for c in cands if c.coverage_center is not None),
        coverage_end=_mean_or_none_round(c.coverage_end for c in cands if c.coverage_end is not None),
        coverage_downstream=_mean_or_none_round(c.coverage_downstream for c in cands if c.coverage_downstream is not None))
    if n_samples != 1:
        call.set_info("STDEV_POS", _stdev(c.pos for c in cands))
        call.set_info("STDEV_LEN", _stdev(c.svlen for c in cands))
    if abs(call.svlen) < config.minsvlen_screen:
        return None
    task.sv_id += 1
    return call


def coverage_rows(sblocks, block_index, config):
    """[n_samples][bins_per_block] int32 of one block: each sample's `_COVERAGE` from the first part of its block (parallel.py:544-545),
    -1 where the sample has no block or no such key.  sblocks: per sample in list order, its parts or None"""
    step = config.coverage_binsize_combine
    per_block = config.snf_block_size // step
    rows = np.full((len(sblocks), per_block), -1, np.int32)
    for si, parts in enumerate(sblocks):
        if parts is None:
            continue
        for k, v in parts[0]["_COVERAGE"].items():
            j = (int(k) - block_index) // step
            if 0 <= j < per_block and (int(k) - block_index) % step == 0:
                rows[si, j] = v
    return rows


@dataclass
class Plan:
    """flat form of every chain of one or more tasks: what snfb_combine_groups reads"""
    cands: list = field(default_factory=list)               # candidate objects in device order
    chains: list = field(default_factory=list)              # (task index, svtype index, cand_off, n_cand, chunk_off, n_chunk)
    chunks: list = field(default_factory=list)              # (cand_off, n_cand, curr_bin, size, cov_block, block position in the task)
    cov_blocks: list = field(default_factory=list)          # block start per coverage row
    cov_rows: list = field(default_factory=list)            # [n_samples][bins_per_block] int32, -1 = no such key
    contig_ids: dict = field(default_factory=dict)


class CombineTask:
    """parallel.CombineTask: same constructor meaning (contig, start, end → block_indices), `execute` returns the calls"""

    def __init__(self, id, contig, start, end, config, sv_id=0, block_indices=None):
        self.id, self.contig, self.start, self.end, self.config, self.sv_id = id, contig, start, end, config, sv_id
        bs = config.snf_block_size
        self.block_indices = list(block_indices) if block_indices is not None else list(range(start, end + bs, bs))     # parallel.py:400-402

    # ---- host: chunks
    def plan(self, readers, plan: Plan, task_index=0):
        cfg = self.config
        bin_min = cfg.combine_min_size
        bin_max = max(25, int(len(cfg.snf_input_info) * 0.5))
        thr = cfg.combine_support_threshold
        ids = [s["internal_id"] for s in cfg.snf_input_info]
        per_type = {t: [] for t in TYPES}                        # chunks of each chain, in block order
        for bpos, block_index in enumerate(self.block_indices):
            sblocks = {sid: readers[sid].read_blocks(self.contig, block_index) for sid in ids}
            if all(b is None for b in sblocks.values()):
                continue
            cov_row = len(plan.cov_blocks)
            plan.cov_blocks.append(block_index)
            plan.cov_rows.append(coverage_rows([sblocks[sid] for sid in ids], block_index, cfg))
            for t in TYPES:
                bins = {}
                for si, sid in enumerate(ids):
                    if sblocks[sid] is None:
                        continue
                    for blk in sblocks[sid]:
                        for cand in blk[t]:
                            if cand.support < thr:
                                continue
                            cand.sample_internal_id = sid
                            cand._sample_index = si
                            bins.setdefault(int(cand.pos / bin_min) * bin_min, []).append(cand)
                if not bins:
                    continue
                size, svcands = 0, []
                order = sorted(bins)
                for b in order:
                    svcands.extend(bins[b])
                    size += bin_min
                    if (not cfg.combine_exhaustive and len(svcands) >= bin_max) or b == order[-1]:
                        svcands = sorted(svcands, key=lambda c: c.support, reverse=True)         # cluster.py:361 (stable)
                        per_type[t].append((svcands, b, size, cov_row, bpos))
                        size, svcands = 0, []
        for ti, t in enumerate(TYPES):
            if not per_type[t]:
                continue
            c0, k0 = len(plan.cands), len(plan.chunks)
            for svcands, b, size, cov_row, bpos in per_type[t]:
                plan.chunks.append((len(plan.cands), len(svcands), b, size, cov_row, bpos))
                plan.cands.extend(svcands)
            plan.chains.append((task_index, ti, c0, len(plan.cands) - c0, k0, len(plan.chunks) - k0))

    # ---- host: SVGroup.call in emission order
    @staticmethod
    def emit(tasks, plan: Plan, out):
        """out: (cand_group, emit_chunk, emit_ord, cov_non) from the device -> calls per task, in the reference's order"""
        result = {}
        for task_index, pairs in CombineTask.emit_batches(tasks, plan, out).items():
            calls = [c for _, c in pairs]
            if not getattr(tasks[task_index].config, "no_sort", False):
                calls.sort(key=lambda c: c.pos)                     # CombineResult.store_calls / finalize (result.py:137-149)
            result[task_index] = calls
        return result

    @staticmethod
    def emit_batches(tasks, plan: Plan, out):
        """out as for `emit` -> per task index, [(batch, call)] in the reference's emission order.  batch: the position of the block whose
        iteration emits the call, which the reference stores as one result.store_calls batch (parallel.py:478-481, 568-569): the chunk's
        block, or the task's last block for the groups kept to the end"""
        cand_group, emit_chunk, emit_ord, cov_non = out
        n_chunk = len(plan.chunks)
        members = {}
        for i, g in enumerate(cand_group.tolist()):
            members.setdefault(g, []).append(i)
        per_task = {}
        for task_index, ti, c0, nc, k0, nk in plan.chains:
            for g in range(c0, c0 + nc):
                ek = int(emit_chunk[g])
                if ek < 0:
                    continue
                # emission order: blocks, then svtypes, then chunks of that (block, svtype), then list order; kept-to-the-end groups last by svtype
                key = (1, ti, 0, int(emit_ord[g])) if ek == n_chunk else (0, plan.chunks[ek][5], ti, ek, int(emit_ord[g]))
                per_task.setdefault(task_index, []).append((key, g))
        result = {}
        for task_index, task in enumerate(tasks):
            ids = [s["internal_id"] for s in task.config.snf_input_info]
            last = len(task.block_indices) - 1
            pairs = []
            for key, g in sorted(per_task.get(task_index, []), key=lambda kg: kg[0]):
                cs = [plan.cands[i] for i in members[g]]
                incl = set(c.sample_internal_id for c in cs)
                cov = {sid: int(cov_non[g, si]) for si, sid in enumerate(ids) if sid not in incl}
                call = call_group(SVGroup(cs, incl, cov), task.config, task)
                if call is not None:
                    pairs.append((last if key[0] == 1 else key[1], call))
            result[task_index] = pairs
        return result

    def execute(self, worker=None, readers=None, ctx=None):
        """parallel.py:443-572; `worker` carries the device context like CallTask's"""
        from . import binding
        cfg = self.config
        own = readers is None
        if own:
            readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in cfg.snf_input_info}
        try:
            plan = Plan()
            self.plan(readers, plan)
            if ctx is None:
                ctx = getattr(worker, "ctx", None) or binding.Context(getattr(worker, "device", 0))
            out = ctx.combine_groups(plan, cfg)
            return CombineTask.emit([self], plan, out)[0]
        finally:
            if own:
                for r in readers.values():
                    r.close()


def plan_arrays(plan: Plan, config):
    """numpy form of a Plan (the snfb_combine_in fields)"""
    n = len(plan.cands)
    pos = np.fromiter((c.pos for c in plan.cands), np.int32, n)
    svlen = np.fromiter((c.svlen for c in plan.cands), np.int32, n)
    sample = np.fromiter((c._sample_index for c in plan.cands), np.uint32, n)
    mate_contig = np.zeros(n, np.int32)
    mate_pos = np.zeros(n, np.int32)
    for i, c in enumerate(plan.cands):
        if c.svtype == "BND":
            mate_contig[i] = plan.contig_ids.setdefault(c.bnd_info.mate_contig, len(plan.contig_ids))
            mate_pos[i] = c.bnd_info.mate_ref_start
    chains = np.array([(c0, nc, k0, nk, 1 if TYPES[ti] == "BND" else 0, 0) for _, ti, c0, nc, k0, nk in plan.chains], np.uint32).reshape(-1, 6)
    chunks = np.array([(c0, nc, b, size, row, 0) for c0, nc, b, size, row, _ in plan.chunks], np.int32).reshape(-1, 6)
    step = config.coverage_binsize_combine
    per_block = config.snf_block_size // step
    cov = np.stack(plan.cov_rows).astype(np.int32) if plan.cov_rows else np.zeros((0, len(config.snf_input_info), per_block), np.int32)
    block_start = np.array(plan.cov_blocks, np.int64)
    alts = [c.alt.encode("latin-1") if isinstance(c.alt, str) else bytes(c.alt or b"") for c in plan.cands]
    alt_len = np.fromiter((len(x) for x in alts), np.uint32, n)
    alt_off = np.zeros(n, np.uint64)
    if n:
        alt_off[1:] = np.cumsum(alt_len[:-1], dtype=np.uint64)
    alt = np.frombuffer(b"".join(alts) + b"\0", np.uint8).copy()
    return dict(alt=alt, alt_off=alt_off, alt_len=alt_len, pos=pos, svlen=svlen, sample=sample, mate_contig=mate_contig, mate_pos=mate_pos, chains=chains, chunks=chunks, cov=np.ascontiguousarray(cov),
                block_start=block_start, bins_per_block=per_block, cov_binsize=step, n_samples=len(config.snf_input_info))
