"""Runs the UNMODIFIED reference (/root/reference/src/sniffles) on a packed record block.

TEST INFRASTRUCTURE ONLY.  It exists to (1) pin the C oracle (oracle/snf_oracle.c) against
the reference itself and (2) generate the committed golden fixtures under tests/golden/
(tests/golden/make_golden.py).  /root/reference does not exist on the GPU box, so nothing
outside this directory and tests/golden/make_golden.py may import this module.

The reference only duck-types its reads (accessor list: SURVEY.md §2), so the records of a
block are exposed as `DuckRead` objects behind a fake `bam.fetch`; pysam is replaced by the
stub in oracle/pyref/stubs.
"""
import os
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REFERENCE_SRC = os.environ.get("SNIFFLES_REFERENCE_SRC", "/root/reference/src")

SEQ_CODE = "=ACMGRSVTWYHKDBN"


def import_reference():
    if not os.path.isdir(REFERENCE_SRC):
        raise RuntimeError(f"reference tree not found at {REFERENCE_SRC}")
    for p in (os.path.join(_HERE, "stubs"), REFERENCE_SRC):
        if p not in sys.path:
            sys.path.insert(0, p)
    import sniffles.config, sniffles.leadprov, sniffles.cluster, sniffles.sv  # noqa
    import sniffles.postprocessing, sniffles.parallel, sniffles.consensus  # noqa
    return sys.modules["sniffles"]


class DuckRead:
    """pysam.AlignedSegment look-alike over one packed record."""
    __slots__ = ("_b", "_i", "_r", "_ct", "_seq", "query_name", "flag", "mapping_quality", "reference_start",
                 "reference_name", "_qas", "_qae", "_rend", "query_length")

    def __init__(self, block, i):
        self._b, self._i = block, i
        r = self._r = block.rec[i]
        self._ct = None
        self._seq = None
        vo, lq = int(r["var_off"]), int(r["l_qname"])
        self.query_name = bytes(block.var[vo:vo + lq]).decode()
        self.flag = int(r["flag"])
        self.mapping_quality = int(r["mapq"])
        self.reference_start = int(r["pos"])
        self.reference_name = block.contig_names[int(block.task[int(r["task"])]["contig"])]
        self.query_length = int(r["l_seq"])
        ct = self.cigartuples
        k, qs = 0, 0
        while k < len(ct) and ct[k][0] in (4, 5):
            if ct[k][0] == 4:
                qs += ct[k][1]
            k += 1
        k, qe = len(ct) - 1, self.query_length
        while k >= 0 and ct[k][0] in (4, 5):
            if ct[k][0] == 4:
                qe -= ct[k][1]
            k -= 1
        self._qas, self._qae = qs, qe
        self._rend = self.reference_start + sum(l for o, l in ct if o in (0, 2, 3, 7, 8))

    @property
    def cigartuples(self):
        if self._ct is None:
            r = self._r
            co, n = int(r["cigar_off"]), int(r["n_cigar"])
            c = self._b.cigar[co:co + n]
            self._ct = [(int(x) & 15, int(x) >> 4) for x in c]
        return self._ct

    is_secondary = property(lambda s: bool(s.flag & 256))
    is_supplementary = property(lambda s: bool(s.flag & 2048))
    is_reverse = property(lambda s: bool(s.flag & 16))
    reference_end = property(lambda s: s._rend)
    reference_length = property(lambda s: s._rend - s.reference_start)
    query_alignment_start = property(lambda s: s._qas)
    query_alignment_end = property(lambda s: s._qae)
    query_alignment_length = property(lambda s: s._qae - s._qas)

    @property
    def query_sequence(self):
        if self._seq is None:
            r = self._r
            so, n = int(r["seq_off"]), int(r["l_seq"])
            raw = np.asarray(self._b.seq[so:so + (n + 1) // 2])
            codes = np.empty(len(raw) * 2, np.uint8)
            codes[0::2] = raw >> 4
            codes[1::2] = raw & 15
            lut = np.frombuffer(SEQ_CODE.encode(), np.uint8)
            self._seq = lut[codes[:n]].tobytes().decode()
        return self._seq

    def has_tag(self, t):
        a = int(self._r["aux_flags"])
        return bool(a & {"NM": 1, "HP": 2, "PS": 4, "SA": 8}.get(t, 0))

    def get_tag(self, t):
        r = self._r
        if not self.has_tag(t):
            raise KeyError(t)
        if t == "NM":
            return int(r["nm"])
        if t == "HP":
            return int(r["hp"])
        if t == "PS":
            return int(r["ps"])
        vo, lq, sl = int(r["var_off"]), int(r["l_qname"]), int(r["sa_len"])
        return bytes(self._b.var[vo + lq:vo + lq + sl]).decode()


class DuckBam:
    def __init__(self, block, task_index):
        self.block, self.t = block, task_index
        self.idx = np.nonzero(block.rec["task"] == task_index)[0]

    def get_reference_length(self, contig):
        return int(self.block.task[self.t]["contig_len"])

    def fetch(self, contig, start, end, until_eof=False):
        for i in self.idx:
            rd = DuckRead(self.block, int(i))
            if rd.reference_start < end and rd.reference_end > start:
                yield rd


def make_config(*extra_args):
    import_reference()
    from sniffles.config import SnifflesConfig
    return SnifflesConfig("--input", "x.bam", "--vcf", "o.vcf", *extra_args)


def run_task(block, t, config, finalize=True):
    """build_leadtab -> call_candidates -> finalize_candidates of the reference on task t.
    Returns a dict: leadtab (dumped before clustering mutates the leads), read_count, mean_nm,
    cands (as they leave call_candidates), final (after finalize_candidates), cov_mean."""
    import_reference()
    from sniffles import leadprov, parallel
    from sniffles.region import Region
    task = block.task[t]
    contig = block.contig_names[int(task["contig"])]
    tr = None
    if int(task["tr_n"]) > 0:
        o, n = int(task["tr_off"]), int(task["tr_n"])
        tr = [(int(block.tr[2 * (o + k)]), int(block.tr[2 * (o + k) + 1])) for k in range(n)]
    if getattr(block, "mask", None) is not None and len(block.mask):
        # --reference: LeadProvider._mask_N_coverage reads the contig through pysam.FastaFile (leadprov.py:420-443)
        import pysam as _stub
        lo, hi = int(block.mask_task_off[t]), int(block.mask_task_off[t + 1])
        runs = [(int(block.mask[2 * m]), int(block.mask[2 * m + 1])) for m in range(lo, hi)]
        clen = int(task["contig_len"])

        class _Fasta:
            def __init__(self, path):
                pass

            def fetch(self, ctg, start=None, end=None):
                seq = bytearray(b"A" * clen)
                for a, b in runs:
                    seq[max(a, 0):min(b, clen)] = b"N" * (min(b, clen) - max(a, 0))
                return bytes(seq[start:end]).decode() if start is not None else bytes(seq).decode()
        _stub.FastaFile = _Fasta
        config.reference = "reference.fa"
    if not hasattr(config, "mode"):
        config.mode = "call_sample"          # set by the CLI driver (sniffles:101-148)
    tk = parallel.CallTask(id=int(task["task_id"]), sv_id=0, contig=contig, start=int(task["start"]),
                           end=int(task["end"]), config=config, tandem_repeats=tr)
    config.task_read_id_offset_mult = 10 ** 9
    tk.lead_provider = leadprov.LeadProvider(config, tk.id * config.task_read_id_offset_mult, contig)
    tk.lead_provider.build_leadtab([Region(contig, tk.start, tk.end)], DuckBam(block, t))
    out = dict(leadtab=leadtab_dump(tk.lead_provider), read_count=tk.lead_provider.read_count,
               mean_nm=float(config.average_regional_nm))
    qc = not (config.snf is not None or config.no_qc)
    cands = tk.call_candidates(qc, config)
    out["cov_mean"] = float(tk.coverage_average_total)
    out["cands"] = [_cand_dict(c, block) for c in cands]
    if finalize:
        final = tk.finalize_candidates(cands, not qc, config)
        out["final"] = [_final_dict(c) for c in final]
        out["vcf"], out["vcf_ref"] = reference_vcf_lines(final, config, None), reference_vcf_lines(final, config, FakeFasta())
    return out


def write_reference_snf(block, config_args, path, reference=None):
    """The reference's own --snf output for a block: every task runs CallTask's SNF branch (parallel.py:279-292: store the candidates,
    annotate_block_coverages, write_and_index) and SNFile.write_results joins the parts (snf.py:193-224).  `reference`: a FASTA path
    for --reference, read through whatever pysam.FastaFile the caller installed (LeadProvider._mask_N_coverage, leadprov.py:420-443)."""
    import io
    import os
    import types
    import_reference()
    from sniffles import leadprov, parallel, snf as refsnf
    from sniffles.region import Region
    config = make_config("--snf", path, *config_args)
    config.reference = reference
    if not hasattr(config, "mode"):
        config.mode = "call_sample"
    config.task_read_id_offset_mult = 10 ** 9
    results = []
    for t in range(len(block.task)):
        task = block.task[t]
        contig = block.contig_names[int(task["contig"])]
        tr = None
        if int(task["tr_n"]) > 0:
            o, n = int(task["tr_off"]), int(task["tr_n"])
            tr = [(int(block.tr[2 * (o + k)]), int(block.tr[2 * (o + k) + 1])) for k in range(n)]
        tk = parallel.CallTask(id=int(task["task_id"]), sv_id=0, contig=contig, start=int(task["start"]), end=int(task["end"]), config=config, tandem_repeats=tr)
        tk.lead_provider = leadprov.LeadProvider(config, tk.id * config.task_read_id_offset_mult, contig)
        tk.lead_provider.build_leadtab([Region(contig, tk.start, tk.end)], DuckBam(block, t))
        cands = tk.call_candidates(False, config)
        tk.finalize_candidates(cands, True, config)
        part = f"{path}.tmp_{tk.id}.snf"
        with open(part, "wb") as handle:
            out = refsnf.SNFile(config, handle)
            for c in cands:
                out.store(c)
            out.annotate_block_coverages(tk.lead_provider)
            out.write_and_index()
        results.append(types.SimpleNamespace(task_id=tk.id, contig=contig, snf_index=out.get_index(), snf_total_length=out.get_total_length(), snf_candidate_count=len(cands),
                                             snf_filename=part, has_snf=True, coverage_average_total=tk.coverage_average_total))
    with open(path, "wb") as handle:
        final = refsnf.SNFile(config, handle)
        for r in results:
            final.add_result(r)
        final.write_results(config, list(block.contig_names))
    return path


class FakeFasta:
    """deterministic reference bases (with a few IUPAC codes) for the VCF writer's REF / anchor fetches; same class feeds both writers"""
    ALPHABET = "ACGTACGTACGTRYNACGTSWK"

    def fetch(self, contig, start=None, end=None):
        if start is None or end is None or start < 0 or end < start:
            raise ValueError("bad interval")
        h = sum(ord(ch) for ch in contig)
        return "".join(self.ALPHABET[(h + 7 * p + (p >> 5)) % len(self.ALPHABET)] for p in range(start, end))


def reference_vcf_lines(final, config, fasta):
    """records the reference's own VCF.write_call emits for the finalized calls (vcf.py:216-350), on deep copies"""
    import copy
    import io
    from sniffles import vcf as refvcf
    if not getattr(config, "sample_ids_vcf", None):
        config.sample_ids_vcf = [(0, "SAMPLE")]
    buf = io.StringIO()
    w = refvcf.VCF(config, buf)
    w.reference_handle = fasta
    for c in final:
        w.write_call(copy.deepcopy(c))
    return buf.getvalue().splitlines()


def lead_tuple(ld):
    b = ld.bnd_info
    return [ld.svtype, ld.ref_start, ld.ref_end, ld.qry_start, ld.qry_end, ld.strand, ld.mapq,
            ld.source, ld.svlen, None if ld.seq is None else len(ld.seq), ld.read_qname, int(ld.hap),
            bool(ld.is_sa), ld.read_len,
            None if b is None else [b.mate_contig, b.mate_ref_start, bool(b.is_first), bool(b.is_reverse)]]


def leadtab_dump(lp):
    """{svtype: [[bin, [lead_tuple...]], ...]} in bin order, leads in reference (BAM) order."""
    out = {}
    for svtype, tab in lp.leadtab.items():
        out[svtype] = [[b, [lead_tuple(ld) for ld in tab[b]]] for b in sorted(tab)]
    return out


def _cand_dict(c, block):
    cl = c.postprocess.cluster
    d = dict(svtype=c.svtype, pos=c.pos, end=c.end, svlen=c.svlen, support=c.support, qual=c.qual,
             precise=bool(c.precise), fwd=c.fwd, rev=c.rev,
             cov=[c.coverage_upstream, c.coverage_start, c.coverage_center, c.coverage_end, c.coverage_downstream],
             stdev_pos=c.info.get("STDEV_POS"), stdev_len=c.info.get("STDEV_LEN"),
             support_long=c.info.get("SUPPORT_LONG"), support_sa=c.info.get("SUPPORT_SA"),
             hap_counts=list(cl.hap_counts), sa_counts=list(cl.sa_counts), id=c.id, cluster_id=cl.id,
             n_leads=len(cl.leads), n_long=len(cl.leads_long) if cl.leads_long else 0,
             leads=[[ld.read_qname, ld.ref_start, ld.svlen, None if ld.seq is None else len(ld.seq)] for ld in cl.leads],
             rnames=sorted(c.rnames), nm=c.nm)
    if c.bnd_info is not None:
        b = c.bnd_info
        d["bnd"] = [b.mate_contig, b.mate_ref_start, bool(b.is_first), bool(b.is_reverse)]
        d["alt"] = c.alt
    return d


def _final_dict(c):
    gt = c.genotypes.get(0)
    return dict(svtype=c.svtype, pos=c.pos, svlen=c.svlen, support=c.support, filter=c.filter, qc=bool(c.qc),
                alt=c.alt, gt=None if gt is None else [gt[0], gt[1], gt[2], gt[3], gt[4], list(gt[5]) if gt[5] else None],
                vaf=c.info.get("VAF"), phase=c.info.get("PHASE"), id=c.id)


def combine_call_dict(c):
    """what a combined call is compared on (both sides build it with this function)"""
    gts = {int(k): [v[0], v[1], v[2], v[3], v[4], list(v[5]) if v[5] else None] + ([v[6]] if len(v) > 6 else []) for k, v in sorted(c.genotypes.items())}
    return dict(contig=c.contig, svtype=c.svtype, pos=c.pos, end=c.end, svlen=c.svlen, id=c.id, alt=c.alt, qual=c.qual, filter=c.filter,
                precise=bool(c.precise), support=c.support, fwd=c.fwd, rev=c.rev, nm=c.nm,
                cov=[c.coverage_upstream, c.coverage_start, c.coverage_center, c.coverage_end, c.coverage_downstream],
                info={k: c.info[k] for k in sorted(c.info)}, genotypes=gts, n_rnames=None if c.rnames is None else len(c.rnames))


def reference_combine(snf_paths, contigs, config_args=()):
    """The reference's own multi-sample combine over SNF files: the setup of sniffles:372-437, then one CombineTask per contig
    (sniffles:466-476) executed in this process (parallel.py:443-572).  Returns (config, {contig: [SVCall]}, vcf_lines)."""
    import_reference()
    from sniffles import parallel, snf as refsnf
    config = make_config(*config_args)
    config.mode = "combine"
    config.input = list(snf_paths)
    config.snf_input_info, config.sample_ids_vcf = [], []
    for k, path in enumerate(snf_paths):
        f = refsnf.SNFile(config, open(path, "rb"), filename=path)
        f.read_header()
        sid = f.header["config"].get("sample_id") or os.path.splitext(os.path.basename(path))[0]
        config.snf_input_info.append({"internal_id": k, "sample_id": sid, "filename": path})
        config.sample_ids_vcf.append((k, sid))
        f.close()
    out, tid = {}, 0
    for name, length in contigs:
        task = parallel.CombineTask(id=tid, contig=name, start=0, end=length - 1, assigned_process_id=None, sv_id=0, config=config, regions=None)
        res = task.execute()
        out[name] = list(res.svcalls) if getattr(res, "svcalls", None) else []
        tid += 1
    lines = reference_vcf_lines([c for name, _ in contigs for c in out[name]], config, FakeFasta())
    return config, out, lines
