"""Host epilogue of the hot path (SURVEY.md §8a row D1): the scalar, per-candidate decisions the
reference makes between clustering and VCF emission — QC filters, support thresholds, phasing
summary and genotype likelihoods.  They stay on the host (O(#candidates), Python floats give
the reference's exact arithmetic); every quantity that needs the leads was already reduced on
the device (snfb_cand: coverage probes, strand count, SA counts, phase aggregates, hap counts).

Behaviour follows /root/reference/src/sniffles/postprocessing.py (qc_sv 200-441, qc_sv_support
133-198, annotate_sv 25-66, qc_sv_post_annotate 444-600, phase_sv 626-654, genotype_sv 607-623),
genotyping.py (62-241) and parallel.py (Task.finalize_candidates 129-201, rescue_phasing 203-249).
The `--dev-filter` accumulation mode is not supported.
"""
import math
from dataclasses import dataclass, field
from typing import Optional

from . import abi

NO_SIZE_TYPES = ("BND", "SINGLE_LEFT", "SINGLE_RIGHT")


@dataclass
class SVCallBNDInfo:                      # sv.py:36-43
    mate_contig: str
    mate_ref_start: int
    is_first: bool
    is_reverse: bool


@dataclass
class ClusterView:
    """What the epilogue still needs to know about a candidate's cluster."""
    n_strands: int
    sa_counts: tuple
    hap_counts: tuple
    lead_qry_start: list                   # only filled in mosaic mode (MOSAIC_SV_CLOSE_EDGE)
    lead_read_len: list
    lead_nm: list                          # only for rescue_phasing
    n_leads: int
    hp_top: int
    hp_support: int
    hp_other: int
    ps_top: Optional[int]
    ps_support: int
    ps_other: int


@dataclass
class SVCall:                              # field surface of sv.SVCall (sv.py:87-131)
    contig: str
    pos: int
    id: str
    ref: str
    alt: str
    qual: int
    filter: str
    info: dict
    svtype: str
    svlen: int
    end: int
    genotypes: dict
    precise: bool
    support: int
    rnames: Optional[list]
    qc: bool
    nm: float
    postprocess: Optional[ClusterView]
    svlens: list = None
    fwd: int = None
    rev: int = None
    coverage_upstream: int = 0
    coverage_downstream: int = 0
    coverage_start: int = 0
    coverage_center: int = 0
    coverage_end: int = 0
    sample_internal_id: int = None
    bnd_info: SVCallBNDInfo = None
    cand_index: int = None                 # index of the device candidate in the run's emission order (force calling maps matches by it)

    def set_info(self, k, v):
        self.info[k] = v

    def get_info(self, k):
        return self.info.get(k)

    def has_info(self, k):
        return k in self.info

    @property
    def is_single_break(self):
        return self.svtype.startswith("SINGLE")

    def finalize(self):
        self.postprocess = None


def calls_from_result(res, task_index, lo, hi, contig_names, task_contig, task_id, config, rec_nm=None, want_leads=False, names=None):
    """snfb_cand[lo:hi] of one task -> SVCall objects as they leave Task.call_candidates (sv.py:561-598).  names: the run's
    binding.ReadNames (--output-rnames), which fill SVCall.rnames; without them rnames stays None."""
    out = []
    rnames = names.per_candidate(res.rn_off, lo, hi) if names is not None else None
    for k, c in enumerate(res.cand[lo:hi]):
        svtype = abi.SVTYPE_NAMES[int(c["svtype"])]
        info = {}
        if svtype == "BND":
            mc = int(c["bnd_mate_contig"])
            mate = contig_names[mc] if mc >= 0 else "?"
            first, rev = bool(c["bnd_is_first"]), bool(c["bnd_is_reverse"])
            br = "]" if rev else "["
            alt = ("N" if first else "") + br + f"{mate}:{int(c['bnd_mate_pos'])}" + br + ("N" if not first else "")     # sv.py:631-635
            bnd = SVCallBNDInfo(mate, int(c["bnd_mate_pos"]), first, rev)
            info["CHR2"] = mate
        else:
            alt, bnd = f"<{svtype}>", None
            if svtype == "INS":
                info["SUPPORT_LONG"] = int(c["support_long"])
            elif svtype == "DEL":
                info["SUPPORT_SA"] = int(c["support_sa"])
        # util.stdev returns the int 0 for fewer than two values (util.py:25-27): a one-lead cluster prints STDEV_POS=0, not 0.000
        one = int(c["fwd"]) + int(c["rev"]) < 2
        info["STDEV_POS"] = 0 if one else float(c["stdev_pos"])
        if not math.isnan(float(c["stdev_len"])):
            info["STDEV_LEN"] = 0 if one else float(c["stdev_len"])
        sa_total = int(c["sa_total"])
        qs, rl, nm = [], [], []
        if want_leads:
            ll = res.cand_leads[int(c["lead_off"]):int(c["lead_off"]) + int(c["lead_n"])]
            qs, rl = [int(x) for x in ll["qry_start"]], [int(x) for x in ll["read_len"]]
            if rec_nm is not None:
                nm = [float(l["nm_sa"]) if (int(l["flags"]) & 7) == abi.BND else float(rec_nm[int(l["rec"])]) for l in ll]
        cv = ClusterView(n_strands=int(c["n_strands"]), sa_counts=(int(c["sa_count"]), int(c["sa_count"]) / float(sa_total) if sa_total else 0.0),
                         hap_counts=tuple(int(x) for x in c["hap_counts"]), lead_qry_start=qs, lead_read_len=rl, lead_nm=nm, n_leads=int(c["lead_n"]),
                         hp_top=int(c["hp_top"]), hp_support=int(c["hp_support"]), hp_other=int(c["hp_other"]),
                         ps_top=None if c["ps_top_null"] else int(c["ps_top"]), ps_support=int(c["ps_support"]), ps_other=int(c["ps_other"]))
        call = SVCall(contig=task_contig, pos=int(c["pos"]), id=f"{svtype}.{k:X}S{task_id:X}", ref="N", alt=alt, qual=int(c["qual"]), filter="PASS",
                      info=info, svtype=svtype, svlen=int(c["svlen"]), end=int(c["end"]), genotypes={}, precise=bool(c["precise"]),
                      support=int(c["support"]), rnames=None if rnames is None else rnames[k], qc=True, nm=float(c["nm_mean"]), postprocess=cv, fwd=int(c["fwd"]), rev=int(c["rev"]),
                      coverage_upstream=int(c["cov_upstream"]), coverage_downstream=int(c["cov_downstream"]), coverage_start=int(c["cov_start"]),
                      coverage_center=int(c["cov_center"]), coverage_end=int(c["cov_end"]), bnd_info=bnd, cand_index=lo + k)
        if svtype == "INS" and int(c["alt_off"]) >= 0 and not config.symbolic:
            call.alt = res.alt[int(c["alt_off"]):int(c["alt_off"]) + int(c["alt_len"])].tobytes().decode()      # annotate_sv, done on the device
        out.append(call)
    return out


# ---------------------------------------------------------------- support thresholds
def rescale_support(call, config):
    if call.svtype != "INS" or call.svlen < config.long_ins_length:
        return call.support
    return round(call.support * (config.long_ins_rescale_base + config.long_ins_rescale_mult * (float(call.svlen) / config.long_ins_length)))


def _nonzero(xs):
    return [x for x in xs if x != 0]


def support_ok(call, coverage_global, config):
    if config.minsupport != "auto":
        return call.support >= config.minsupport
    cov = _nonzero([call.coverage_upstream, call.coverage_downstream]) or _nonzero([call.coverage_start, call.coverage_center, call.coverage_end])
    regional = coverage_global
    if cov:
        regional = round(sum(cov) / len(cov)) or coverage_global
    w = config.minsupport_auto_regional_coverage_weight
    blended = regional * w + coverage_global * (1.0 - w)
    return rescale_support(call, config) >= round(config.minsupport_auto_base + config.minsupport_auto_mult * blended)


def qc_sv_support(call, coverage_global, config):
    if support_ok(call, coverage_global, config):
        return True
    call.filter = "SUPPORT_MIN"
    return False


# ---------------------------------------------------------------- pre-annotation QC
def _cov_change(call, sign, scaled):
    """COV_CHANGE_DEL (sign=+1) / COV_CHANGE_DUP (sign=-1) tests of qc_sv."""
    u, c, d = call.coverage_upstream, call.coverage_center, call.coverage_downstream
    central = c > (u + d) * scaled if sign > 0 else c < (u + d) * scaled
    if central:
        if u > c > d:
            if d / u < 0.7:
                return True
        elif u < c < d:
            if u / d < 0.7:
                return True
    if sign > 0 or central:       # the DUP variant nests the slope tests under the central test
        if u > d:
            if 0.5 > d / u or (c > d if sign > 0 else c < d):
                return True
        elif u < d:
            if 0.5 > u / d or (u < c if sign > 0 else u > c):
                return True
    return False


def qc_sv(call, config):
    def fail(name):
        call.filter = name
        return False

    sized = call.svtype not in NO_SIZE_TYPES
    if config.qc_stdev:
        sp = call.get_info("STDEV_POS")
        if sp > config.qc_stdev_abs_max:
            return fail("STDEV_POS")
        if sized and sp / abs(call.svlen) > 2.0:
            return fail("STDEV_POS")
        sl = call.get_info("STDEV_LEN")
        if sl is not None and sl != 0:
            if call.svtype != "BND" and sl / abs(call.svlen) > 1.0:
                return fail("STDEV_LEN")
            if sl > config.qc_stdev_abs_max:
                return fail("STDEV_LEN")
    if call.is_single_break and not config.dev_output_candidates:
        return fail("SINGLE_BREAK")
    if abs(call.svlen) < config.minsvlen and call.svtype != "BND" and (call.support < 10 or config.minsvlen_hard_cap):
        return fail("SVLEN_MIN")
    if call.svtype == "BND" and config.qc_bnd_filter_strand and call.postprocess.n_strands < 2:
        return fail("STRAND_BND")
    if (call.svtype == "DEL" and config.long_del_length != -1 and abs(call.svlen) >= config.long_del_length and not config.mosaic
            and abs(call.svlen) <= config.dev_longer_del):
        if _cov_change(call, +1, config.long_del_coverage / 2.0):
            return fail("COV_CHANGE_DEL")
    elif (call.svtype == "DUP" and config.long_dup_length != -1 and abs(call.svlen) >= config.long_dup_length and not config.mosaic
          and abs(call.svlen) <= config.dev_longer_dup):
        if _cov_change(call, -1, config.long_dup_coverage / 2.0):
            return fail("COV_CHANGE_DUP")
    elif call.svtype == "INS" and (call.coverage_upstream < config.qc_coverage or call.coverage_downstream < config.qc_coverage):
        return fail("COV_CHANGE_INS")
    if call.svtype in ("INS", "DEL"):
        sa_inline, sap_inline = call.postprocess.sa_counts
        sa_split = call.info.get("SUPPORT_SA")
        if sap_inline > config.dev_inline_sa_support_max and sa_inline > 5 and (sa_split == 0 or sa_split is None):
            return fail("INLINE_SA")
    call.set_info("COVERAGE_VAR", None)        # the forward-difference sampler is never fed in the reference
    frac = config.qc_coverage_max_change_frac
    if frac != -1.0:
        vals = [float(v) if v != 0 else 1.0 for v in (call.coverage_upstream, call.coverage_start, call.coverage_center, call.coverage_end, call.coverage_downstream)]
        for (a, b), name in zip(zip(vals, vals[1:]), ("US", "SC", "CE", "ED")):
            if abs(a - b) / max(a, b) > frac:
                return fail("COV_CHANGE_FRAC_" + name)
    return True


# ---------------------------------------------------------------- phasing and genotypes
def phase_sv(call, config):
    cv = call.postprocess
    hp, ps = str(cv.hp_top), ("NULL" if cv.ps_top is None else str(cv.ps_top))
    hp_f = "PASS" if (float(cv.hp_other) / (cv.hp_support + cv.hp_other) < config.phase_conflict_threshold and hp != "NULL" and cv.hp_support > 0) else "FAIL"
    ps_f = "PASS" if (float(cv.ps_other) / (cv.ps_support + cv.ps_other) < config.phase_conflict_threshold and ps != "NULL" and cv.ps_support > 0) else "FAIL"
    call.set_info("PHASE", f"{hp},{ps},{cv.hp_support},{cv.ps_support},{hp_f},{ps_f}")
    return (hp if hp in config.phase_identifiers and hp_f == "PASS" else None), (ps if ps_f == "PASS" else None)


class _NoGenotype(Exception):
    pass


def _mean_nonzero(values):
    vals = [v for v in values if v != 0]
    if not vals:
        raise _NoGenotype()
    return round(sum(vals) / len(vals))


def _gt_support_and_coverage(call, config):
    t = call.svtype
    if t == "INS":
        return rescale_support(call, config), lambda s: _mean_nonzero([call.coverage_center])
    if t == "DUP":
        return call.support, lambda s: _mean_nonzero([call.coverage_start, call.coverage_end]) + round(s * 0.75)
    if t == "INV":
        return call.support, lambda s: _mean_nonzero([call.coverage_upstream, call.coverage_downstream]) + round(s * 0.5)
    if t == "DEL" and call.get_info("SUPPORT_SA"):
        sa = call.get_info("SUPPORT_SA")
        return call.support, lambda s: _mean_nonzero([call.coverage_start + sa, call.coverage_center + sa, call.coverage_end + sa])
    return call.support, lambda s: _mean_nonzero([call.coverage_start, call.coverage_center, call.coverage_end])


def _binom(k, n, p):
    try:
        return (p ** k) * ((1.0 - p) ** (n - k))
    except OverflowError:
        return 1.0


def _lr(q1, q2):
    if q1 / q2 > 0:
        try:
            return math.log(q1 / q2, 10)
        except ValueError:
            return 0
    return 0


def genotype_sv(call, config, phase):
    support, cov_fn = _gt_support_and_coverage(call, config)
    try:
        coverage = cov_fn(support)
    except _NoGenotype:
        call.filter, call.qc = "GT_FAILED", False
        return
    coverage = max(coverage, support)
    af = support / float(coverage)
    top = max(support, coverage)
    ns, nc = (round(support * (250 / float(top))), round(coverage * (250 / float(top)))) if top > 250 else (support, coverage)
    lik = [((0, 0), _binom(ns, nc, config.genotype_error)), ((0, 1), _binom(ns, nc, 1.0 / config.genotype_ploidy)), ((1, 1), _binom(ns, nc, 1.0 - config.genotype_error))]
    lik.sort(key=lambda kv: kv[1], reverse=True)
    total = sum(q for _, q in lik)
    lik = [(gt, q / total) for gt, q in lik]
    (gt1, q1), (_, q2) = lik[0], lik[1]
    qz = [q for gt, q in lik if gt == (0, 0)][0]
    z = min(60, int(-10 * _lr(qz, q1)))
    gq = min(60, int(-10 * _lr(q2, q1)))
    keep_dup = call.svtype == "DUP" and af >= config.dev_min_dup_vaf
    z_filter = z < config.genotype_min_z_score and not config.mosaic
    if z_filter and call.svtype == "INS" and call.svlen >= config.long_ins_length and config.detect_large_ins:
        z_filter = False
    if call.filter == "PASS" and z_filter:
        call.filter = "PASS" if keep_dup else "GT"
        call.qc = not config.pass_only
    a, b = (0, 1) if keep_dup and gt1 == (0, 0) else gt1
    call.genotypes[0] = (a, b, gq, coverage - support, support, phase)
    call.set_info("VAF", af)
    # hom-alt calls skip the haplotype filter (postprocessing.py:612-623)
    if a == b == 1 and call.get_info("PHASE"):
        hp, ps, hs, pss, _hf, pf = call.get_info("PHASE").split(",")
        if hp != "0":
            call.genotypes[0] = (a, b, gq, coverage - support, support, (hp, ps))
            call.set_info("PHASE", f"{hp},{ps},{hs},{pss},PASS,{pf}")


def annotate_sv(call, config):
    phase = phase_sv(call, config) if config.phase else (None, None)
    genotype_sv(call, config, phase)
    # the INS ALT sequence was computed on the device (snfb_consensus) and is already in call.alt


# ---------------------------------------------------------------- post-annotation QC
def qc_sv_post_annotate(call, config, coverage_total):
    def fail(name):
        call.filter = name
        return False

    af = call.get_info("VAF") or 0
    mosaic_sv = af <= config.mosaic_af_max
    gt = call.genotypes.get(0)
    if (call.coverage_center < config.qc_coverage and (gt is None or (gt[0] != "." and gt[0] + gt[1] < 2))
            and call.svtype != "DEL" and abs(call.svlen) > config.long_del_length):
        return fail("COV_MIN_GT")
    if config.mosaic and not mosaic_sv and not qc_sv_support(call, coverage_total, config):
        return False
    qc_nm = config.mosaic_qc_nm if (config.mosaic and mosaic_sv) else config.qc_nm
    if qc_nm and call.nm > config.qc_nm_threshold * config.qc_nm_mult and (gt is None or gt[1] == 0):
        return fail("ALN_NM")
    if not config.mosaic and mosaic_sv and not (call.svtype == "DUP" and af >= config.dev_min_dup_vaf):
        return fail("MOSAIC_VAF")
    if config.mosaic and mosaic_sv:
        sp, sl = call.info.get("STDEV_POS"), call.info.get("STDEV_LEN")
        need = config.mosaic_min_reads
        if sp is not None and sl is not None and call.svtype in ("INS", "DEL", "DUP", "INV", "BND"):
            svlen_info = call.info.get("SVLEN", 1)
            low = (not call.precise or sl / abs(call.svlen) > 0.1 or sp > 5) and abs(svlen_info) <= config.max_svlen_mosaic
            need = config.mosaic_min_reads if (call.svtype in ("BND", "INV") or low) else config.mosaic_min_reads - 1
        if call.support < need:
            return fail("SUPPORT_MIN")
        if call.svtype != "BND" and abs(call.svlen) > config.max_svlen_mosaic:
            return fail("SVLEN_MAX_MOSAIC")
    if call.svtype != "BND":
        long_ins = call.svtype == "INS" and call.svlen >= config.long_ins_length
        one_strand = call.postprocess.n_strands < 2
        if not (config.mosaic and mosaic_sv) and config.qc_strand:
            if not long_ins and one_strand:
                return fail("STRAND")
        elif (config.mosaic and mosaic_sv) and config.mosaic_qc_strand:
            if not long_ins and one_strand and call.support >= config.mosaic_use_strand_thresholds:
                return fail("STRAND_MOSAIC")
    if config.mosaic and mosaic_sv and call.svtype in ("INV", "DUP") and call.svlen < config.mosaic_qc_invdup_min_length:
        return fail("SVLEN_MIN_MOSAIC")
    if call.coverage_center < config.qc_coverage and call.svtype not in ("DEL", "INS"):
        # sic: `(svtype == "INV" and svlen) > long_inv_length` in the reference (postprocessing.py:555)
        inv_term = call.svlen if call.svtype == "INV" else False
        if not (inv_term > config.long_inv_length and not (config.mosaic and mosaic_sv)):
            return fail("COV_MIN")
    if config.mosaic:
        if mosaic_sv and (af < config.mosaic_af_min or af > config.mosaic_af_max):
            return fail("MOSAIC_VAF")
        if not mosaic_sv and not config.mosaic_include_germline:
            return fail("NOT_MOSAIC_VAF")
        if mosaic_sv and call.svtype not in NO_SIZE_TYPES:
            cv = call.postprocess
            d = config.dev_min_close_edge_dist
            close = sum(1 for q, rl in zip(cv.lead_qry_start, cv.lead_read_len) if q <= d or abs(rl - q) <= d)
            if float(close) / call.support >= config.dev_min_read_close_edge_prop:
                return fail("MOSAIC_SV_CLOSE_EDGE")
    return True


def rescue_phasing(call, config, min_in_phase=0.75, min_reads=3):
    """Task.rescue_phasing (parallel.py:203-249): un-filter MOSAIC_VAF calls that are well phased."""
    if config.mode != "call_sample":
        return False
    cv = call.postprocess
    import numpy as np
    sv_nm = float(np.nanmean(cv.lead_nm)) if cv.lead_nm else float("nan")
    if sv_nm > config.genotype_error or cv.n_leads <= min_reads or "PHASE" not in call.info:
        return False
    hp, _, _, _, hp_filter, _ = call.info["PHASE"].split(",")
    if hp_filter != "PASS":
        return False
    hp = int(hp)
    _, sv1, sv2, _, hap1, hap2 = cv.hap_counts
    if hp == 1:
        every, sv = hap1, sv1
    elif hp == 2:
        every, sv = hap2, sv2
    else:
        return False
    if every == 0:
        return False
    if float(sv) / float(every) >= min_in_phase and call.filter == "MOSAIC_VAF":
        a, _b, gq, dr, dv, p = call.genotypes[0]
        call.filter, call.genotypes[0], call.qc = "PASS", (a, 1, gq, dr, dv, p), True
        return True
    return False


def finalize_candidates(calls, keep_qc_fails, config, coverage_total):
    """Task.finalize_candidates (parallel.py:129-201) without the --dev-locasm-do branch."""
    for call in calls:
        call.qc = call.qc and qc_sv(call, config)
        if not config.mosaic and call.qc:
            call.qc = call.qc and qc_sv_support(call, coverage_total, config)
        annotate_sv(call, config)
        call.qc = call.qc and qc_sv_post_annotate(call, config, coverage_total)
        rescue_ok = call.svtype != "BND" and abs(call.svlen) <= config.dev_maxsvlen_extra and call.support >= int(config.dev_minreads_extra * 0.60)
        if config.phase and not call.qc and rescue_ok:
            try:
                rescue_phasing(call, config)
            except Exception:
                pass
        call.finalize()
    return calls
