"""Force calling (`--genotype-vcf`): the SVs of an input VCF genotyped in one sample (sniffles:191-214, 289-358; parallel.py:300-369;
vcf.py:352-478; result.py:118-130).

  * `read_targets` is VCF.read_svs_iter: the same parsing steps, so every error names the same line with the same message.  A `.gz`
    input is read as BGZF text (bamio.BgzfReader), where the reference goes through pysam.VariantFile (DESIGN §4);
  * `plan` makes one task per processed contig, [0, contig_len - 1), holding the contig's targets with start <= pos < end;
  * matching and the coverage probes run on the device (snfb_genotype_targets); `genotype_of` and the rewrite stay on the host;
  * `genotype_vcf(config)` drives the mode in the device passes of call.call_sample (call.device_passes): the tasks with targets, in
    task-id order, grouped so that their inflated BAM bytes fit a budget (host memory holds one pass's BGZF bytes).  A pass is
    call.load_pass (N mask, snfb_load_bam, snfb_run), one snfb_genotype_targets call for the targets of its tasks, then its tasks'
    records, rewritten through vcf.open_output, before the next pass loads.  The records come in task order, and in target-file
    order inside a task, so the output is the same at every budget.  The genotype step's device memory (about 63 bytes per target
    and 28 per candidate of the pass, kept on the context) sits inside the margin call.device_budget leaves (DESIGN §8)."""
import io
import logging
import os
import time
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import abi, bamio, binding, vcf

log = logging.getLogger("sniffles_b200.genotype")

SVTYPE_CODE = {name: code for code, name in enumerate(abi.SVTYPE_NAMES[:5])}      # sv.TYPES: INS DEL DUP INV BND


class TargetVcfError(ValueError):
    """a malformed target VCF (the reference's util.fatal_error while parsing)"""


@dataclass
class TargetBnd:
    mate_contig: str
    mate_ref_start: int
    is_first: bool
    is_reverse: bool


@dataclass
class Target:
    """the fields of sv.SVCall that force calling reads or writes"""
    contig: str
    pos: int
    id: int
    ref: str
    alt: str
    qual: Optional[int]
    filter: str
    info: dict
    svtype: object = None
    svlen: int = None
    end: int = None
    bnd_info: TargetBnd = None
    raw_vcf_line: str = None
    raw_vcf_line_index: int = None
    genotype_match_sv: object = None
    coverage_start: int = 0
    coverage_center: int = 0
    coverage_end: int = 0
    genotypes: dict = None


def _lines(path):
    ext = os.path.splitext(path)[1].lower()
    if ext == ".vcf":
        with open(path, "r") as f:
            yield from f
    elif ext == ".gz":
        r = bamio.BgzfReader(path)
        try:
            chunks, v = [], 0
            while True:
                data, v = r.read_from(v, 1 << 22)
                if not data:
                    break
                chunks.append(data)
        finally:
            r.close()
        yield from io.StringIO(b"".join(chunks).decode("utf-8"), newline=None)
    else:
        raise TargetVcfError("Expected a .vcf or .vcf.gz file for genotyping using --genotype-vcf")


def read_targets(path):
    """(header text, [Target]) of a VCF, parsed as VCF.read_svs_iter parses it (vcf.py:352-428)"""
    header, out, line_index = [], [], 0
    for line in _lines(path):
        try:
            line_index += 1
            line_strip = line.strip()
            if line_strip == "" or line_strip[0] == "#":        # a blank line raises IndexError here, as in the reference
                if line_strip[0] == "#":
                    header.append(line_strip + "\n")
                continue
            CHROM, POS, _, REF, ALT, QUAL, FILTER, INFO = line.split("\t")[:8]
            info_dict = {}
            for info_item in INFO.split(";"):
                if "=" in info_item:
                    key, value = info_item.split("=")
                else:
                    key, value = info_item, True
                info_dict[key] = value
            call = Target(contig=CHROM, pos=int(POS) - 1, id=line_index, ref=REF, alt=ALT, qual=int(QUAL) if QUAL != "." else None,
                          filter=FILTER, info=info_dict)
            if len(call.alt) > len(call.ref):
                call.svtype, call.svlen, call.end = "INS", len(call.alt), call.pos
            else:
                call.svtype, call.svlen = "DEL", -len(call.ref)
                call.end = call.pos + call.svlen
            if "SVTYPE" in info_dict:
                call.svtype = info_dict["SVTYPE"]
                if call.svtype == "TRA":
                    call.svtype = "BND"
            if "SVLEN" in info_dict:
                call.svlen = int(info_dict["SVLEN"])
            if "END" in info_dict:
                call.end = int(info_dict["END"])
            if call.svtype == "BND":
                bnd_parts = call.alt.replace("]", "[").split("[")
                if len(bnd_parts) > 2:
                    mate_contig, mate_ref_start = bnd_parts[1].split(":")
                    call.bnd_info = TargetBnd(mate_contig, int(mate_ref_start), call.alt[0] == "N", "]" in call.alt)
                else:
                    raise ValueError("BND ALT not formatted according to VCF 4.2 specifications")
            call.raw_vcf_line = line_strip
            call.raw_vcf_line_index = line_index
            out.append(call)
        except Exception as e:
            raise TargetVcfError(f"Error parsing input VCF: Line {line_index}: {e}") from e
    return "".join(header), out


def rewrite_header(orig_header, config):
    """VCF.rewrite_header_genotype (vcf.py:449-478): the text written before the records"""
    header_lines = orig_header.split("\n")
    header_lines.insert(1, '##genotypeFileDate="' + str(getattr(config, "start_date", "")) + '"')
    header_lines.insert(1, '##genotypeCommand="' + str(getattr(config, "command", "")) + '"')
    header_lines.insert(1, f"##genotypeSource={getattr(config, 'version', 'Sniffles2')}_{getattr(config, 'build', 'b200')}")
    have = {k: any("##FORMAT=<ID=" + k + "," in h for h in header_lines) for k in ("GT", "GQ", "DR", "DV")}
    for k, t, d in (("GT", "String", "Genotype"), ("GQ", "Integer", "Genotype quality"), ("DR", "Integer", "Number of reference reads"),
                    ("DV", "Integer", "Number of variant reads")):
        if not have[k]:
            header_lines.insert(len(header_lines) - 2, f'##FORMAT=<ID={k},Number=1,Type={t},Description="{d}">')
    return "\n".join(header_lines)


def genotype_of(target, config):
    """the genotype written for a target (parallel.py:349-361, vcf.py:430-441): the matched candidate's, else one from the coverage"""
    m = target.genotype_match_sv
    if m is not None and len(m.genotypes) > 0:
        return m.genotypes[0]
    coverage = round(sum([target.coverage_start, target.coverage_center, target.coverage_end]) / 3)
    return (0, 0, 0, coverage, 0, (None, None)) if coverage > 0 else config.genotype_none


def rewrite_line(target, config):
    """VCF.rewrite_genotype (vcf.py:430-447): FORMAT without :PS, the sample column with PS when phased, as the reference writes them"""
    return "\t".join(target.raw_vcf_line.split("\t")[:8] + [config.genotype_format, vcf.format_genotype(genotype_of(target, config), config.phase)])


def plan(contigs, targets, config):
    """the task plan of tasks.plan (one task per processed contig, sniffles:289-358) with each task's targets: [(task id, contig, start,
    end, [Target])], a task holding the targets of its contig with start <= pos < end"""
    from . import tasks
    by_contig = {}
    for t in targets:
        by_contig.setdefault(t.contig, []).append(t)
    return [(tid, name, s, e, [t for t in by_contig.get(name, []) if s <= t.pos < e]) for tid, name, s, e in tasks.plan(contigs, config)[1]]


def encode(targets, task_index, name_to_id):
    """SoA columns of snfb_gt_in for one task's targets"""
    n = len(targets)
    cols = {k: np.zeros(n, "<i4") for k in ("task", "svtype", "pos", "svlen", "bnd_is_first", "mate_contig")}
    cols["task"][:] = task_index
    for i, t in enumerate(targets):
        for k, v in (("pos", t.pos), ("svlen", t.svlen)):
            if not -2**31 <= v < 2**31:
                raise TargetVcfError(f"Error parsing input VCF: Line {t.raw_vcf_line_index}: {k} {v} does not fit 32 bits")
        cols["svtype"][i] = SVTYPE_CODE.get(t.svtype, -1) if isinstance(t.svtype, str) else -1
        cols["pos"][i], cols["svlen"][i] = t.pos, t.svlen
        if t.bnd_info is not None:
            cols["bnd_is_first"][i] = int(t.bnd_info.is_first)
            cols["mate_contig"][i] = name_to_id.get(t.bnd_info.mate_contig, -1)
        else:
            cols["mate_contig"][i] = -1
    return cols


def device_targets(ctx, per_task, name_to_id, config):
    """ONE snfb_genotype_targets call for the targets of several tasks of the block on `ctx`: per_task = [(task index, [Target])] in task
    order.  Returns {task index: (match, cov_start, cov_center, cov_end, bnd_no_prev) sliced to that task's targets}"""
    parts = [encode(ts, k, name_to_id) for k, ts in per_task]
    keys = ("task", "svtype", "pos", "svlen", "bnd_is_first", "mate_contig")
    cols = [np.concatenate([p[k] for p in parts]) if parts else np.zeros(0, "<i4") for k in keys]
    res = ctx.genotype_targets(*cols, config.combine_match, config.combine_match_max)
    out, o = {}, 0
    for k, ts in per_task:
        out[k] = tuple(a[o:o + len(ts)] for a in res)
        o += len(ts)
    return out


def write_tasks(handle, br, jobs, config):
    """GenotypeTask.execute for every job [(task id, contig, start, end, [Target], block task index)] of the block run `br` (its
    br.genotype filled by device_targets), the records written in task order as GenotypeResult.emit writes them; a failing task is
    logged and left out, as the reference's worker leaves it out.  Returns the number of records written."""
    from . import tasks
    written = 0
    for tid, name, s, e, ts, k in jobs:
        task = tasks.GenotypeTask(id=tid, sv_id=0, contig=name, start=s, end=e, config=config, genotype_svs=ts, block_run=br, task_index=k)
        try:
            done, _ = task.execute()
        except tasks.GenotypeTaskError as err:
            task.log_failure(log, err)
            continue
        for t in done:
            handle.write(rewrite_line(t, config) + "\n")
            written += 1
    return written


def genotype_vcf(config, device=0, budget=None, stats=None):
    """the --genotype-vcf run mode: config.input (one indexed BAM) and config.genotype_vcf -> config.vcf.  Returns the number of records
    written.  budget: the inflated BAM bytes one device pass may load (default: call.device_budget).  stats: a dict that receives the
    run's split, with call.call_sample's keys where they apply (passes, pass_inflated_bytes, load_bam_s and run_s per pass, read_s,
    index_s, wall_s) and parse_s (the target VCF), genotype_s (per pass, the snfb_genotype_targets round trip) and write_s (the tasks'
    host epilogue and rewrite, the header and the output's close: a .vcf.gz is compressed and indexed then)."""
    from . import call, tasks
    st = stats if stats is not None else {}
    t0 = time.perf_counter()
    header, targets = read_targets(config.genotype_vcf)
    log.info(f"Opening for reading: {config.genotype_vcf} (read {len(targets)} SVs to be genotyped)")
    st.update(passes=0, pass_inflated_bytes=[], load_bam_s=[], run_s=[], genotype_s=[], read_s=0.0, write_s=0.0, parse_s=time.perf_counter() - t0)
    t1 = time.perf_counter()
    path = config.input[0] if isinstance(config.input, (list, tuple)) else config.input
    bam = call.open_indexed(path)
    planned, targets_of = [], {}
    for tid, name, s, e, ts in plan(bam.contigs, targets, config):
        if not ts:                                      # a task without targets writes nothing
            continue
        try:
            tasks.fetch_windows(name, s, e, config.regions_by_contig.get(name))
        except ValueError as err:                       # the task fails in the reference's worker: its targets are not written
            tasks.GenotypeTask(tid, 0, name, s, e, config).log_failure(log, err)
            continue
        planned.append((tid, name, s, e))
        targets_of[tid] = ts
    tr_all = tasks.load_tandem_repeats(config.tandem_repeats, config.tandem_repeat_region_pad) if config.tandem_repeats else {}
    ctx = tasks.device_context(device)
    if budget is None:
        budget = call.device_budget(device)
    st["index_s"] = time.perf_counter() - t1
    written = 0
    with vcf.open_output(config, ctx) as handle:
        t1 = time.perf_counter()
        handle.write(rewrite_header(header, config))
        st["write_s"] += time.perf_counter() - t1
        # a pass's targets are matched against the candidates and coverage of the block resident on the context: every step of a pass
        # ends before the next pass loads
        for group, br in call.device_passes(ctx, bam, planned, config, tr_all, budget, st):
            t1 = time.perf_counter()
            try:
                br.genotype = device_targets(ctx, [(k, targets_of[it.id]) for k, it in enumerate(group)], bam.name_to_id, config)
            except binding.SnfbError as e:
                names = ", ".join(it.contig for it in group)
                raise call.CallSampleError(f"the target genotyping of the device pass over contig(s) {names} "
                                           f"({st['pass_inflated_bytes'][-1]} inflated BAM bytes) failed: {e}") from e
            t2 = time.perf_counter()
            written += write_tasks(handle, br, [(it.id, it.contig, it.start, it.end, targets_of[it.id], k) for k, it in enumerate(group)], config)
            st["genotype_s"].append(t2 - t1)
            st["write_s"] += time.perf_counter() - t2
        t1 = time.perf_counter()
    st["write_s"] += time.perf_counter() - t1
    bam.close()
    st["wall_s"] = time.perf_counter() - t0
    return written
