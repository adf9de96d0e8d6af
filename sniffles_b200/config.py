"""Host-side mirror of the reference's `SnifflesConfig` object surface (config.py:103-619):
same attribute names, defaults and derived constants, so code written against the reference's
config namespace (Task, QC, genotyping, writers) runs unchanged.  Table-driven rather than a
copy of the reference's argparse set-up; only flags that reach the hot path, the QC/genotype
epilogue or the writers are declared."""
import argparse
import logging
import os
import tempfile

log = logging.getLogger(__name__)


def _bed_region(line):
    """(contig, start, end) of a BED line's first three tab-separated fields; ValueError when they are missing or not integers"""
    fields = line.split("\t")
    if len(fields) < 3:
        raise ValueError(f"{len(fields)} tab-separated field(s), 3 needed")
    return fields[0], int(fields[1]), int(fields[2])


def _string_region(text):
    """(contig, start, end) of `contig:start-end`; ValueError for any other shape"""
    parts = text.split(":")
    if len(parts) != 2:
        raise ValueError("expected one ':'")
    bounds = parts[1].split("-")
    if len(bounds) != 2:
        raise ValueError("expected one '-'")
    return parts[0], int(bounds[0]), int(bounds[1])


def regions_by_contig(config):
    """the regions of --regions (a BED file; lines starting with '#' and blank lines skipped) or, without it, of the --region strings:
    {contig: [(contig, start, end), ...]} in input order, never sorted or merged.  An entry that does not parse is skipped with a warning;
    a missing BED file raises FileNotFoundError; --contig together with --regions exits.  Pinned against the reference's parser by
    tests/golden/regions/expected.json."""
    if config.contig and config.regions:
        raise SystemExit("Please provide either --contig or --regions, not both.")
    if config.regions is not None:
        with open(config.regions, "r") as f:
            entries = [(line, _bed_region) for line in f.readlines() if not line.startswith("#") and line.strip() != ""]
    else:
        entries = [(text, _string_region) for text in config.region or []]
    out = {}
    for text, parse in entries:
        try:
            r = parse(text)
        except ValueError as e:
            log.warning(f"skipping region {text!r}: {e}")
            continue
        out.setdefault(r[0], []).append(r)
    return out


def _tobool(v):
    if isinstance(v, bool):
        return v
    s = str(v).strip().lower()
    if s in ("true", "t", "1", "yes", "y"):
        return True
    if s in ("false", "f", "0", "no", "n"):
        return False
    raise argparse.ArgumentTypeError("Boolean value (True | False) required for argument")


# (flag(s), kwargs) — defaults are the reference's (config.py:173-446)
_OPTIONS = [
    (("-i", "--input"), dict(type=str, nargs="+", required=True)),
    (("-v", "--vcf"), dict(type=str, default=None)),
    (("--snf",), dict(type=str, default=None)),
    (("--reference",), dict(type=str, default=None)),
    (("--phase",), dict(action="store_true", default=argparse.SUPPRESS)),
    (("-t", "--threads"), dict(type=int, default=4)),
    (("-c", "--contig"), dict(type=str, default=None, action="append")),
    (("--regions",), dict(type=str, default=None)),
    (("--region",), dict(type=str, default=None, action="append")),
    (("--tmp-dir",), dict(type=str, default="")),
    (("--all-contigs",), dict(action="store_true", default=False)),
    (("--minsupport",), dict(type=str, default="3")),
    (("--minsupport-auto-mult",), dict(type=float, default=None)),
    (("--minsvlen",), dict(type=str, default="~50")),
    (("--minsvlen-screen-ratio",), dict(type=float, default=0.9)),
    (("--mapq",), dict(type=int, default=argparse.SUPPRESS)),
    (("--no-qc", "--qc-output-all"), dict(action="store_true", default=False)),
    (("--pass-only",), dict(action="store_true", default=False)),
    (("--qc-stdev",), dict(type=_tobool, default=True)),
    (("--qc-stdev-abs-max",), dict(type=int, default=500)),
    (("--qc-strand",), dict(type=_tobool, default=False)),
    (("--qc-coverage",), dict(type=int, default=1)),
    (("--long-ins-length",), dict(type=int, default=2500)),
    (("--long-del-length",), dict(type=int, default=50000)),
    (("--long-inv-length",), dict(type=int, default=10000)),
    (("--long-del-coverage",), dict(type=float, default=0.66)),
    (("--long-dup-length",), dict(type=int, default=50000)),
    (("--long-dup-coverage",), dict(type=float, default=1.33)),
    (("--qc-bnd-filter-strand",), dict(type=_tobool, default=True)),
    (("--bnd-min-split-length",), dict(type=int, default=1000)),
    (("--max-splits-kb",), dict(type=float, default=0.1)),
    (("--max-splits-base",), dict(type=int, default=3)),
    (("--min-alignment-length",), dict(type=int, default=argparse.SUPPRESS)),
    (("--phase-conflict-threshold",), dict(type=float, default=0.1)),
    (("--detect-large-ins",), dict(type=_tobool, default=True)),
    (("--max-unknown-pct",), dict(type=float, default=0.5)),
    (("--large-coverage-sample-interval",), dict(type=int, default=5000)),
    (("--cluster-binsize",), dict(type=int, default=100)),
    (("--cluster-r",), dict(type=float, default=2.5)),
    (("--cluster-repeat-h",), dict(type=float, default=1.5)),
    (("--cluster-repeat-h-max",), dict(type=float, default=1000)),
    (("--cluster-merge-pos",), dict(type=int, default=150)),
    (("--cluster-merge-len",), dict(type=float, default=0.22)),
    (("--cluster-merge-bnd",), dict(type=int, default=1000)),
    (("--genotype-ploidy",), dict(type=int, default=2)),
    (("--genotype-error",), dict(type=float, default=0.05)),
    (("--sample-id",), dict(type=str, default=None)),
    (("--genotype-vcf",), dict(type=str, default=None)),
    (("--output-rnames",), dict(action="store_true", default=False)),
    (("--no-consensus",), dict(action="store_true", default=False)),
    (("--no-sort",), dict(action="store_true", default=False)),
    (("--no-progress",), dict(action="store_true", default=False)),
    (("--quiet",), dict(action="store_true", default=False)),
    (("--max-del-seq-len",), dict(type=int, default=50000)),
    (("--symbolic",), dict(action="store_true", default=False)),
    (("--allow-overwrite",), dict(action="store_true", default=False)),
    (("--mosaic",), dict(action="store_true", default=False)),
    (("--mosaic-af-max",), dict(type=float, default=0.218)),
    (("--mosaic-af-min",), dict(type=float, default=0.05)),
    (("--mosaic-qc-invdup-min-length",), dict(type=int, default=500)),
    (("--mosaic-qc-nm",), dict(action="store_true", default=True)),
    (("--mosaic-qc-nm-mult",), dict(type=float, default=1.66)),
    (("--mosaic-qc-coverage-max-change-frac",), dict(type=float, default=-1)),
    (("--mosaic-qc-strand",), dict(type=_tobool, default=True)),
    (("--mosaic-include-germline",), dict(action="store_true", default=False)),
    (("--max-svlen-mosaic",), dict(type=int, default=50000)),
    (("--tandem-repeats",), dict(type=str, default=None)),
    (("--dev-emit-sv-lengths",), dict(action="store_true", default=False)),
    (("--dev-keep-lowqual-splits",), dict(action="store_true", default=False)),
    (("--dev-seq-cache-maxlen",), dict(type=int, default=50000)),
    (("--consensus-max-reads",), dict(type=int, default=20)),
    (("--consensus-max-reads-bin",), dict(type=int, default=10)),
    (("--dev-no-resplit",), dict(action="store_true", default=False)),
    (("--dev-no-resplit-repeat",), dict(action="store_true", default=False)),
    (("--repeat",), dict(action="store_true", default=False)),
    (("--qc-nm",), dict(action="store_true", default=False)),
    (("--qc-nm-mult",), dict(type=float, default=1.66)),
    (("--qc-coverage-max-change-frac",), dict(type=float, default=-1)),
    (("--coverage-updown-bins",), dict(type=int, default=5)),
    (("--coverage-shift-bins",), dict(type=int, default=3)),
    (("--cluster-binsize-combine-mult",), dict(type=int, default=5)),
    (("--cluster-resplit-binsize",), dict(type=int, default=20)),
    (("--dev-no-qc",), dict(action="store_true", default=False)),
    (("--dev-filter",), dict(action="store_true", default=False)),
    (("--exclude-flags", "--excl-flags", "-F"), dict(type=int, default=None)),
    (("--dev-output-candidates",), dict(type=str, default=None)),
    (("--dev-single-break-count",), dict(type=int, default=3)),
    (("--dev-single-break-dist",), dict(type=int, default=50)),
    (("--dev-min-leads-cluster",), dict(type=int, default=-1)),
    (("--dev-min-dup-vaf",), dict(type=float, default=1 / 6.0)),
    (("--dev-longer-del",), dict(type=int, default=200000)),
    (("--dev-longer-dup",), dict(type=int, default=200000)),
    (("--dev-minreads-extra",), dict(type=int, default=5)),
    (("--dev-maxsvlen-extra",), dict(type=int, default=10000)),
    (("--dev-locasm-skip-mosaic",), dict(action="store_true", default=False)),
    (("--dev-locasm-do",), dict(action="store_true", default=False)),
    (("--dev-inline-sa-support-max",), dict(type=float, default=0.80)),
    (("--dev-min-close-edge-dist",), dict(type=int, default=500)),
    (("--dev-min-read-close-edge-prop",), dict(type=float, default=0.75)),
    (("--combine-high-confidence",), dict(type=float, default=0.0)),           # multi-sample arguments, config.py:297-312
    (("--combine-low-confidence",), dict(type=float, default=0.2)),
    (("--combine-low-confidence-abs",), dict(type=int, default=2)),
    (("--combine-null-min-coverage",), dict(type=int, default=5)),
    (("--combine-match",), dict(type=int, default=250)),
    (("--combine-match-max",), dict(type=int, default=1000)),
    (("--combine-separate-intra",), dict(action="store_true", default=False)),
    (("--combine-output-filtered",), dict(action="store_true", default=False)),
    (("--combine-pair-relabel",), dict(action="store_true", default=False)),
    (("--combine-pair-relabel-threshold",), dict(type=int, default=20)),
    (("--combine-pctseq",), dict(type=float, default=0.7)),
    (("--combine-support-threshold",), dict(type=int, default=3)),
    (("--combine-consensus",), dict(action="store_true", default=False)),
    (("--combine-max-inmemory-results",), dict(type=int, default=20)),
    (("--combine-population",), dict(type=str, default=None)),
    (("--re-qc",), dict(type=str, default="auto")),
    (("--dev-skip-snf-validation",), dict(action="store_true", default=False)),
    (("--dev-population-snf",), dict(type=str, default=None)),
    (("--dev-combine-medians",), dict(action="store_true", default=False)),
    (("--gpus",), dict(type=int, default=1)),          # new: number of GPUs to shard contigs over
]


class SnifflesConfig(argparse.Namespace):
    """Same attribute surface as the reference's config namespace."""
    GLOBAL = None
    phase = True                       # class default, as in the reference (config.py:147)
    mosaic_min_reads = 3
    mosaic_use_strand_thresholds = 10
    default_cluster_merge_len = 0.22
    default_cluster_merge_len_mosaic = 0.27

    def __init__(self, *args):
        super().__init__()
        p = argparse.ArgumentParser(prog="sniffles", add_help=True)
        for flags, kw in _OPTIONS:
            p.add_argument(*flags, **kw)
        p.parse_args(args=list(args), namespace=self)
        if not self.tmp_dir or not os.path.exists(self.tmp_dir):
            self.tmp_dir = tempfile.gettempdir()
        self.task_count_multiplier = 0
        self.regions_by_contig = regions_by_contig(self)
        # --minsvlen: "~N" = soft cap (config.py:507-517)
        ms = str(self.minsvlen)
        self.minsvlen_hard_cap = not ms.startswith("~")
        self.minsvlen = int(ms.lstrip("~"))
        self.minsvlen_screen = int(self.minsvlen_screen_ratio * self.minsvlen)
        if self.minsupport != "auto":
            self.minsupport = int(self.minsupport)
        if self.dev_no_qc:
            self.no_qc = True
        if not hasattr(self, "mapq"):
            self.mapq = 0 if self.dev_no_qc else 20
        if not hasattr(self, "min_alignment_length"):
            self.min_alignment_length = 0 if self.dev_no_qc else 1000
        self.minsupport_auto_base = 1.5
        self.minsupport_auto_regional_coverage_weight = 0.75
        if self.minsupport_auto_mult is None:
            self.minsupport_auto_mult = 0.1
        self.coverage_binsize = self.cluster_binsize
        self.coverage_binsize_combine = self.cluster_binsize * self.cluster_binsize_combine_mult
        self.consensus_min_reads = 4
        self.consensus_kmer_len = 6
        self.consensus_kmer_skip_base = 3
        self.consensus_kmer_skip_seqlen_mult = 1.0 / 500.0
        self.long_ins_rescale_base = 1.66
        self.long_ins_rescale_mult = 0.33
        self.dev_longer_dup = min(self.long_dup_length * 4, self.dev_longer_dup)
        self.dev_longer_del = min(self.long_del_length * 4, self.dev_longer_del)
        self.bnd_cluster_length = 1000
        self.genotype_format = "GT:GQ:DR:DV"
        self.genotype_none = (".", ".", 0, 0, 0, (None, None))
        self.genotype_null = (0, 0, 0, 0, 0, (None, None))
        self.genotype_min_z_score = 5
        if self.genotype_ploidy != 2:
            raise SystemExit("Currently only --genotype-ploidy 2 is supported")
        self.snf_block_size = 10 ** 5
        self.combine_exhaustive = False                 # config.py:576-580
        self.combine_relabel_rare = False
        self.combine_overlap_abs = 2500
        self.combine_min_size = 100
        self.precise = 25
        self.tandem_repeat_region_pad = 500
        self.id_prefix = "Sniffles2."
        self.phase_identifiers = ["1", "2"]
        if self.mosaic_include_germline:
            self.mosaic = True
        self.qc_nm_measure = self.qc_nm
        if self.mosaic:
            self.qc_nm_measure = self.qc_nm_measure or self.mosaic_qc_nm
            if self.cluster_merge_len == self.default_cluster_merge_len:
                self.cluster_merge_len = self.default_cluster_merge_len_mosaic
        if self.dev_min_leads_cluster == -1:
            self.dev_min_leads_cluster = 1 if self.no_qc else 2
        self.mode = "call_sample" if self.genotype_vcf is None else "genotype_vcf"
        if self.mode != "call_sample" and self.snf is not None:
            raise SystemExit(f"--snf cannot be used with run mode {self.mode}")
        self.qc_nm_threshold = 0.0
        self.average_regional_nm = 0.0
        self.dev_trace_read = False
        self.task_read_id_offset_mult = 10 ** 9
        SnifflesConfig.GLOBAL = self

    @property
    def sort(self):
        return bool(self.vcf_output_bgz) or not self.no_sort

    @property
    def vcf_output_bgz(self):
        if self.vcf:
            return os.path.splitext(self.vcf)[1] in (".gz", ".bgz")
        return None


def default_config(*extra) -> SnifflesConfig:
    return SnifflesConfig("--input", "input.bam", "--vcf", "out.vcf", *extra)
