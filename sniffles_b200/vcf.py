"""VCF emission of finished calls — the writer side of SURVEY.md §8(f)4, restating the observable behaviour of the
reference's `VCF.write_header` / `VCF.write_call` (/root/reference/src/sniffles/vcf.py:120-350) on this package's
`postprocess.SVCall` objects:

  * DEL end rewritten to pos + |svlen| for precise calls (vcf.py:225-226), POS clamped to >= 1 (:223);
  * INS: SVLEN is rewritten to len(ALT) when a sequence is reported, and the call is dropped when that falls below
    --minsvlen (vcf.py:259-264);
  * INFO order PRECISE/IMPRECISE, MOSAIC, then SVTYPE, SVLEN, END, SUPPORT, RNAMES, COVERAGE, STRAND (, NM), then the
    call's own info keys sorted (vcf.py:266-296); floats as %.3f, True as a bare flag (:25-35);
  * DEL REF fetch / INS + BND anchor base from the reference FASTA when one is given, and the IUPAC clean-up that — as in
    the reference — only happens inside the "reference given and REF still N" branch (vcf.py:299-342): bug-compatible;
  * QUAL clamped to 0..60 (:344).

The FASTA reader is any object with `fetch(contig, start, end) -> str` (pysam.FastaFile duck type); none is needed for
symbolic / sequence-free output.  Genotype columns follow format_genotype (vcf.py:50-79)."""
import io
import logging
from collections import Counter

from . import bamio

log = logging.getLogger("sniffles_b200.vcf")

AMBIGUOUS = str.maketrans("RYSWKMBDHV", "N" * 10)          # util.py:169-170

FILTERS = [("PASS", "All filters passed"), ("GT", "Genotype filter"), ("SUPPORT_MIN", "Minimum read support filter"),
           ("STDEV_POS", "SV Breakpoint standard deviation filter"), ("STDEV_LEN", "SV length standard deviation filter"),
           ("COV_MIN", "Minimum coverage filter"), ("COV_MIN_GT", "Minimum coverage filter (missing genotype)"),
           ("COV_CHANGE_DEL", "Coverage change filter for DEL"), ("COV_CHANGE_DUP", "Coverage change filter for DUP"),
           ("COV_CHANGE_INS", "Coverage change filter for INS"),
           ("COV_CHANGE_FRAC_US", "Coverage fractional change filter: upstream-start"), ("COV_CHANGE_FRAC_SC", "Coverage fractional change filter: start-center"),
           ("COV_CHANGE_FRAC_CE", "Coverage fractional change filter: center-end"), ("COV_CHANGE_FRAC_ED", "Coverage fractional change filter: end-downstream"),
           ("COV_VAR", "Coverage variance exceeded"), ("MOSAIC_VAF", "Mosaic variant allele fraction filter"),
           ("NOT_MOSAIC_VAF", "Variant allele fraction filter for non-mosaic"), ("ALN_NM", "Length adjusted mismatch filter"),
           ("STRAND_BND", "Strand support filter for BNDs"), ("STRAND", "Strand support filter for germline SVs"),
           ("STRAND_MOSAIC", "Strand support filter for mosaic SVs"), ("SVLEN_MIN", "SV length filter"),
           ("SVLEN_MIN_MOSAIC", "SV length filter for mosaic SVs (min)"), ("SVLEN_MAX_MOSAIC", "SV length filter for mosaic SVs (max)"),
           ("SINGLE_BREAK", "A single break point was detected but not classified as an SV."),
           ("INLINE_SA", "INLINE/CIGAR-based SV is mostly supported by SA reads"),
           ("MOSAIC_SV_CLOSE_EDGE", "For mosaic SVs, the location is close to the end of the read (either end)"),
           ("GT_FAILED", "Sniffles was unable to genotype this call.")]

INFOS = [("PRECISE", "0", "Flag", "Structural variation with precise breakpoints"), ("IMPRECISE", "0", "Flag", "Structural variation with imprecise breakpoints"),
         ("MOSAIC", "0", "Flag", "Structural variation classified as putative mosaic"), ("SVLEN", "1", "Integer", "Length of structural variation"),
         ("SVTYPE", "1", "String", "Type of structural variation"), ("CHR2", "1", "String", "Mate chromsome for BND SVs"),
         ("SUPPORT", "1", "Integer", "Number of reads supporting the structural variation"),
         ("SUPPORT_INLINE", "1", "Integer", "Number of reads supporting an INS/DEL SV (non-split events only)"),
         ("SUPPORT_SA", "1", "Integer", "Number of reads supporting a DEL SV through supplementary alignments (split events)"),
         ("SUPPORT_LONG", "1", "Integer", "Number of soft-clipped reads putatively supporting the long insertion SV"),
         ("END", "1", "Integer", "End position of structural variation"), ("STDEV_POS", "1", "Float", "Standard deviation of structural variation start position"),
         ("STDEV_LEN", "1", "Float", "Standard deviation of structural variation length"),
         ("COVERAGE", ".", "Float", "Coverages near upstream, start, center, end, downstream of structural variation"),
         ("STRAND", "1", "String", "Strands of supporting reads for structural variant"), ("AC", ".", "Integer", "Allele count, summed up over all samples"),
         ("SUPP_VEC", "1", "String", "List of read support for all samples"),
         ("CONSENSUS_SUPPORT", "1", "Integer", "Number of reads that support the generated insertion (INS) consensus sequence"),
         ("RNAMES", ".", "String", "Names of supporting reads (if enabled with --output-rnames)"), ("VAF", "1", "Float", "Variant Allele Fraction"),
         ("COVERAGE_VAR", "1", "Float", "Variance of coverage across large events"),
         ("NM", ".", "Float", "Mean number of query alignment length adjusted mismatches of supporting reads"),
         ("PHASE", ".", "String", "Phasing information derived from supporting reads, represented as list of: HAPLOTYPE,PHASESET,HAPLOTYPE_SUPPORT,PHASESET_SUPPORT,HAPLOTYPE_FILTER,PHASESET_FILTER"),
         ("LASM", "0", "Flag", "Local assembly used to detect the structural variant")]


def _fmt_info(key, value):
    if isinstance(value, float):
        return f"{key}={value:.3f}"
    if isinstance(value, list):
        return f"{key}={','.join(value)}"
    if value is None:
        value = "."
    if value is True:
        return key
    return f"{key}={value}"


def _phase_parts(phase):
    try:
        hp, ps = phase
    except TypeError:
        hp, ps = (None, ".") if phase is None else (phase, ".")
    return hp, (ps if ps is not None and ps != "NULL" else ".")


def format_genotype(gt, phased):
    """GT:GQ:DR:DV[:PS][:ID] column of one sample (vcf.py:50-79); 7-tuples carry the per-sample SV id of combine mode."""
    svid = None
    if len(gt) == 6:
        a, b, qual, dr, dv, phase = gt
    else:
        a, b, qual, dr, dv, phase, svid = gt
    hp, ps = _phase_parts(phase)
    sep = "/"
    if hp is not None and (a, b) in ((0, 1), (1, 1)) and phased:
        sep = "|"
        if hp == "1":
            a, b = b, a
    cols = [f"{a}{sep}{b}", str(qual), str(dr), str(dv)]
    if phased:
        cols.append(str(ps))
    if svid is not None:
        cols.append(str(svid))
    return ":".join(cols)


class VCFWriter:
    def __init__(self, config, handle, reference=None):
        self.config, self.handle, self.reference = config, handle, reference
        self.call_count = 0
        self.info_order = ["SVTYPE", "SVLEN", "END", "SUPPORT", "RNAMES", "COVERAGE", "STRAND"]
        if getattr(config, "qc_nm_measure", False):
            self.info_order.append("NM")
        if getattr(config, "dev_emit_sv_lengths", False):
            self.info_order.append("SVLENGTHS")
        self.phased = bool(getattr(config, "phase", False))
        self.genotype_format = getattr(config, "genotype_format", "GT:GQ:DR:DV") + (":PS" if self.phased else "")
        self.default_genotype = tuple(getattr(config, "genotype_none", (".", ".", 0, 0, 0, (None, None))))
        if getattr(config, "mode", "call_sample") == "combine":
            self.genotype_format += ":ID"
            self.default_genotype += ("NULL",)
        self.samples = list(getattr(config, "sample_ids_vcf", None) or [(0, "SAMPLE")])

    def _line(self, text):
        self.handle.write(text)
        self.handle.write("\n")

    def write_header(self, contigs_lengths):
        c = self.config
        h = ["fileformat=VCFv4.2", f"source={getattr(c, 'version', 'Sniffles2')}_{getattr(c, 'build', 'b200')}",
             'command="' + str(getattr(c, "command", "")) + '"', 'fileDate="' + str(getattr(c, "start_date", "")) + '"']
        h += [f"contig=<ID={name},length={length}>" for name, length in contigs_lengths]
        h += [f'ALT=<ID={k},Description="{d}">' for k, d in (("INS", "Insertion"), ("DEL", "Deletion"), ("DUP", "Duplication"), ("INV", "Inversion"), ("BND", "Breakend; Translocation"))]
        h += [f'FORMAT=<ID={k},Number=1,Type={t},Description="{d}">' for k, t, d in (
            ("GT", "String", "Genotype"), ("GQ", "Integer", "Genotype quality"), ("DR", "Integer", "Number of reference reads"), ("DV", "Integer", "Number of variant reads"),
            ("PS", "Integer", "Phase-block, zero if none or not phased"), ("ID", "String", "Individual sample SV ID for multi-sample output"))]
        h += [f'FILTER=<ID={k},Description="{d}">' for k, d in FILTERS]
        for k, n, t, d in INFOS:
            h.append(f'INFO=<ID={k},Number={n},Type={t},Description="{d}">')
            if k == "SVLEN" and getattr(c, "dev_emit_sv_lengths", False):
                h.append('INFO=<ID=SVLENGTHS,Number=.,Type=Integer,Description="Lengths of structural variation (all)">')
        if getattr(c, "combine_population", None):
            h.append('INFO=<ID=POPULATION_AF,Number=1,Type=Float,Description="Population Allele Frequency">')
            h.append('INFO=<ID=POPULATION_SIZE,Number=1,Type=Integer,Description="Size of genotyped population for this variant">')
            if getattr(c, "mode", None) == "combine" and self.phased:        # vcf.py:201-204
                log.warning("Sniffles does not provide population phasing, it just displays the phasing information from each independent "
                            "sample. Multi-sample phased genotypes may be inconsistent with population phasing")
        for line in h:
            self._line("##" + line)
        self._line("#CHROM\tPOS\tID\tREF\tALT\tQUAL\tFILTER\tINFO\tFORMAT\t" + "\t".join(name for _, name in self.samples))

    def write_call(self, call) -> int:
        """one VCF record; returns 1 when a line was written (vcf.py:216-350).  Mutates the call like the reference does."""
        c = self.config
        if call.is_single_break:
            return 0
        pos = call.pos if call.pos > 0 else 1
        end = pos + abs(call.svlen) if (call.precise and call.svtype == "DEL") else call.end
        # genotype columns, allele count, support vector
        ac, supvec, cols = 0, [], []
        for internal_id, _ in self.samples:
            gt = call.genotypes.get(internal_id) if call.genotypes else None
            if gt is not None:
                cols.append(format_genotype(gt, self.phased))
                has = gt[0] != "." and gt[4] > 0
                if has:
                    ac += sum(gt[:2])
                supvec.append("1" if has else "0")
            else:
                cols.append(format_genotype(self.default_genotype, self.phased))
                supvec.append("0")
        if len(self.samples) > 1:
            call.set_info("AC", ac)
            call.set_info("SUPP_VEC", "".join(supvec))
            if int("".join(supvec)) == 0:
                return 0
            if ac == 0:
                call.filter = "GT"
        symbolic = bool(getattr(c, "symbolic", False))
        if call.svtype == "INS":
            if call.svlen != len(call.alt) and not symbolic and call.alt != "<INS>":
                call.svlen = len(call.alt)                   # SVLEN follows the reported sequence
            if call.svlen < c.minsvlen:
                return 0
        fields = {"SVTYPE": call.svtype, "SVLEN": call.svlen, "SVLENGTHS": ",".join(map(str, call.svlens)) if call.svlens else None, "END": end,
                  "SUPPORT": call.support, "RNAMES": call.rnames if getattr(c, "output_rnames", False) else None,
                  "COVERAGE": f"{call.coverage_upstream},{call.coverage_start},{call.coverage_center},{call.coverage_end},{call.coverage_downstream}",
                  "STRAND": ("+" if call.fwd > 0 else "") + ("-" if call.rev > 0 else ""), "NM": call.nm}
        if call.svtype == "BND":
            fields["SVLEN"] = fields["SVLENGTHS"] = fields["END"] = None
        parts = ["PRECISE" if call.precise else "IMPRECISE"]
        vaf = call.get_info("VAF")
        if (vaf if vaf is not None else 0) <= c.mosaic_af_max and c.mosaic:
            parts.append("MOSAIC")
        parts += [_fmt_info(k, fields[k]) for k in self.info_order if fields[k] is not None]
        parts += [_fmt_info(k, call.info[k]) for k in sorted(call.info) if call.info[k] is not None]
        ref = self.reference
        if not symbolic and call.svtype == "DEL" and ref is not None and abs(call.svlen) <= getattr(c, "max_del_seq_len", 50000):
            try:
                call.ref = ref.fetch(call.contig, call.pos - 1, call.pos - call.svlen)       # the base before the deletion + the deleted bases
                call.alt = call.ref[0]
            except (KeyError, ValueError):
                call.ref, call.alt = "N", f"<{call.svtype}>"
            else:
                if "N" in call.ref and Counter(call.ref)["N"] / len(call.ref) > getattr(c, "max_unknown_pct", 1.0):
                    return 0
        if symbolic:
            call.ref = "N"
            if call.svtype != "BND":
                call.alt = f"<{call.svtype}>"
        elif ref is not None and call.ref == "N":
            try:
                start = max(0, call.pos - 1)
                call.ref = ref.fetch(call.contig, start, start + 1)
            except (KeyError, ValueError):
                pass
            else:
                if call.svtype == "INS" and call.alt != "<INS>":
                    call.alt = call.ref + call.alt
                elif call.svtype == "BND" and call.alt != "<BND>":
                    call.alt = (call.ref + call.alt[1:]) if call.alt.startswith("N") else call.alt[:-1] + call.ref
            call.ref = call.ref.translate(AMBIGUOUS)         # only on this branch, as in the reference (vcf.py:340-342)
            call.alt = call.alt.translate(AMBIGUOUS)
        call.qual = max(0, min(60, call.qual)) if call.qual is not None else None
        self._line("\t".join(str(v) for v in [call.contig, pos, getattr(c, "id_prefix", "Sniffles2.") + call.id, call.ref, call.alt,
                                             call.qual if call.qual is not None else ".", call.filter, ";".join(parts), self.genotype_format] + cols))
        self.call_count += 1
        return 1


def reference_intervals(calls, config):
    """every (contig, start, end) `VCFWriter.write_call` can fetch from the reference for these calls (vcf.py:304-338): the DEL's anchor
    base plus deleted bases (pos - 1, pos - svlen), and the anchor base (max(0, pos - 1), + 1) of any call.  A superset: what the writer
    skips (symbolic output, long DELs, single breaks) is listed anyway, so one Reference.prefetch serves a whole call set."""
    out = []
    for call in calls:
        if call.svtype == "DEL":
            out.append((call.contig, call.pos - 1, call.pos - call.svlen))
        a = max(0, call.pos - 1)
        out.append((call.contig, a, a + 1))
    return out


class BgzfIndexedOutput:
    """Text handle for a `--vcf out.vcf.gz` (sniffles:229-244, :573-584): VCFWriter writes into it unchanged; `close()` compresses the
    text into BGZF members with `compress(bytes) -> (members, coffsets)` (binding.Context.deflate_bgzf on the product path), then writes
    `path` (members + the BGZF EOF marker) and `path + ".tbi"` (bamio.tabix_index, compressed the same way) — the pair
    `pysam.tabix_index(..., preset="vcf")` leaves.  When the index refuses the text (unsorted lines, a reappearing contig, a position
    beyond 2^29) the ValueError propagates and neither file is written."""

    def __init__(self, path, compress):
        self.path, self.compress = path, compress
        self._buf = io.StringIO()

    def write(self, text):
        return self._buf.write(text)

    def close(self):
        if self._buf is None:
            return
        text = self._buf.getvalue().encode()
        self._buf = None
        z, coffsets = self.compress(text)
        tbi, _ = self.compress(bamio.tabix_index(text, coffsets))
        with open(self.path, "wb") as f:
            f.write(z + bamio._BGZF_EOF)
        with open(self.path + ".tbi", "wb") as f:
            f.write(tbi + bamio._BGZF_EOF)

    def __enter__(self):
        return self

    def __exit__(self, exc_type, exc, tb):
        if exc_type is None:
            self.close()


def open_output(config, ctx):
    """the handle VCFWriter writes `config.vcf` through: a plain text file, or for a .gz / .bgz name (config.vcf_output_bgz) a
    BgzfIndexedOutput compressed on the device of `ctx` (sniffles:250, :575-583)"""
    if not config.vcf_output_bgz:
        return open(config.vcf, "w")
    return BgzfIndexedOutput(config.vcf, ctx.deflate_bgzf)
