"""Force calling (`--genotype-vcf`): the SVs of an input VCF genotyped in one sample (sniffles:191-214, 289-358; parallel.py:300-369;
vcf.py:352-478; result.py:118-130).

  * `read_targets` is VCF.read_svs_iter: the same parsing steps, so every error names the same line with the same message.  A `.gz`
    input is read as BGZF text (bamio.BgzfReader), where the reference goes through pysam.VariantFile (DESIGN §4);
  * `plan` makes one task per processed contig, [0, contig_len - 1), holding the contig's targets with start <= pos < end;
  * matching and the coverage probes run on the device (snfb_genotype_targets); `genotype_of` and the rewrite stay on the host;
  * `genotype_vcf(config)` drives the mode: one device ingest and run for every task, one snfb_genotype_targets call for every target,
    then the rewritten VCF through vcf.open_output."""
import io
import logging
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np

from . import abi, bamio, vcf

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
            log.error(f"Error in worker process while executing {task.label()}: {err}")
            continue
        for t in done:
            handle.write(rewrite_line(t, config) + "\n")
            written += 1
    return written


def genotype_vcf(config, device=0):
    """the --genotype-vcf run mode: returns the number of records written to config.vcf"""
    from . import tasks
    header, targets = read_targets(config.genotype_vcf)
    log.info(f"Opening for reading: {config.genotype_vcf} (read {len(targets)} SVs to be genotyped)")
    path = config.input[0] if isinstance(config.input, (list, tuple)) else config.input
    bam = bamio.BamFile(path)
    planned = []
    for p in plan(bam.contigs, targets, config):
        if not p[4]:                                    # a task without targets writes nothing
            continue
        tid, name, s, e, _ = p
        regions = config.regions_by_contig.get(name)
        try:
            windows = tasks.fetch_windows(name, s, e, regions)
        except ValueError as err:                       # the task fails in the reference's worker: its targets are not written
            log.error(f"Error in worker process while executing GenotypeTask(id={tid}, contig={name}, start={s}, end={e}): {err}")
            continue
        planned.append((p, windows if regions else None))
    tr_all = tasks.load_tandem_repeats(config.tandem_repeats, config.tandem_repeat_region_pad) if config.tandem_repeats else {}
    ctx = tasks.device_context(device)
    with vcf.open_output(config, ctx) as handle:
        handle.write(rewrite_header(header, config))
        if not planned:
            return 0
        tr = {k: [(int(a), int(b)) for a, b in tr_all[p[1]]] for k, (p, _) in enumerate(planned) if p[1] in tr_all}
        # a task with regions: its records carry their region's window, its own bounds only clip the N mask (clipped to the regions here)
        bounds = [(0, bam.get_reference_length(p[1])) if rg else (p[2], p[3]) for p, rg in planned]
        block = bamio.pack_records(bam.contigs, [], [(bam.name_to_id[p[1]], a, b, p[0]) for (p, _), (a, b) in zip(planned, bounds)], tandem_repeats=tr or None)
        # target coverage is N-masked as in GenotypeTask's LeadProvider; without regions the call is the one it always was
        mask_regions = {k: rg for k, (_, rg) in enumerate(planned) if rg}
        tasks.mask_block(block, config, ctx, mask_regions) if mask_regions else tasks.mask_block(block, config, ctx)
        ctx.set_config(abi.Config.from_sniffles(config))
        by_task = [(k, rg or [(p[2], p[3])]) for k, (p, rg) in enumerate(planned)]
        queries, tags, n = [], [], 0
        for (k, w), (p, _) in zip(by_task, planned):
            queries += [(p[1], a, b) for a, b in w]
            tags += [(k, n + g) for g in range(len(w))]
            n += len(w)
        has_regions = any(rg for _, rg in planned)
        bgzf, spans = bam.device_input(queries, tags=tags)
        ctx.set_regions(tasks.region_table(by_task) if has_regions else None)
        n_rec = ctx.load_bam(bgzf, spans, block)["n_rec"]
        res = ctx.run(want_leads=True, want_cands=True, want_seqs=True)
        rec_nm = abi.view(res._rec_nm_ptr, "<f8", n_rec).copy() if getattr(res, "_rec_nm_ptr", None) else None
        br = tasks.BlockRun(block, res, tasks.cand_ranges(res.cand, len(block.task)), rec_nm)
        br.genotype = device_targets(ctx, [(k, p[4]) for k, (p, _) in enumerate(planned)], bam.name_to_id, config)
        return write_tasks(handle, br, [p + (k,) for k, (p, _) in enumerate(planned)], config)
