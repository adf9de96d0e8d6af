"""SNF container — SURVEY.md §8(f)2: the per-sample candidate store the reference writes with --snf and reads back in combine
mode (/root/reference/src/sniffles/snf.py:91-267).

Format (restated): one JSON header line {"config": ..., "index": {contig: {block: [(offset, length), ...]}},
"snf_candidate_count": n}, then gzip(pickle(block)) members back to back (offsets relative to the end of the header line).  A block
holds the candidates of one 100-kb window (config.snf_block_size) as {svtype: [SVCall, ...] for the five SV types} plus
"_COVERAGE": {position: rounded mean coverage of a coverage_binsize_combine window}.

The pickled candidates ARE part of the format: the reference unpickles them as `sniffles.sv.SVCall` (with `SVCallBNDInfo` and
`ForwardDifferenceWelford` inside), so this module pickles and unpickles through classes registered under exactly those module /
class names (`compat_classes`).  When the real `sniffles` package is importable its own classes are used instead."""
import gzip
import importlib
import json
import pickle
import sys
import types
from dataclasses import dataclass, field, fields

TYPES = ["INS", "DEL", "DUP", "INV", "BND"]          # sv.py:31


def compat_classes():
    """(SVCall, SVCallBNDInfo, ForwardDifferenceWelford) under the module path the SNF pickles name"""
    try:
        m = importlib.import_module("sniffles.sv")
        if not getattr(m, "_snfb_shim", False):
            return m.SVCall, m.SVCallBNDInfo, m.ForwardDifferenceWelford
        return m.SVCall, m.SVCallBNDInfo, m.ForwardDifferenceWelford
    except Exception:
        pass
    pkg = types.ModuleType("sniffles")
    pkg.__path__ = []
    mod = types.ModuleType("sniffles.sv")
    mod._snfb_shim = True

    class ForwardDifferenceWelford:                  # sv.py:49-80 (state only: n, m1, m2, last)
        def __init__(self):
            self.n, self.m1, self.m2, self.last = 0, 0, 0, None

    @dataclass
    class SVCallBNDInfo:
        mate_contig: str
        mate_ref_start: int
        is_first: bool
        is_reverse: bool

    @dataclass
    class SVCall:                                    # field set and order of sv.py:87-131
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
        rnames: object
        qc: bool
        nm: float
        postprocess: object
        svlens: list = None
        fwd: int = None
        rev: int = None
        forward_difference_sampler: object = field(default_factory=ForwardDifferenceWelford)
        coverage_upstream: int = 0
        coverage_downstream: int = 0
        coverage_start: int = 0
        coverage_center: int = 0
        coverage_end: int = 0
        sample_internal_id: int = None
        bnd_info: object = None
        support_inline: int = None
        support_splits: int = None
        raw_vcf_line: object = None
        raw_vcf_line_index: object = None

        def set_info(self, k, v):
            self.info[k] = v

        def get_info(self, k):
            return self.info.get(k)

    for cls in (ForwardDifferenceWelford, SVCallBNDInfo, SVCall):
        cls.__module__, cls.__qualname__ = "sniffles.sv", cls.__name__
        setattr(mod, cls.__name__, cls)
    mod.TYPES = list(TYPES)
    pkg.sv = mod
    sys.modules.setdefault("sniffles", pkg)
    sys.modules["sniffles.sv"] = mod
    return SVCall, SVCallBNDInfo, ForwardDifferenceWelford


def population_class():
    """sniffles.snfp.PopulationVariant (snfp.py:25-37), the class a population SNF's blocks pickle: the reference's own when it imports,
    else a dataclass registered under that module path"""
    compat_classes()
    try:
        m = importlib.import_module("sniffles.snfp")
        return m.PopulationVariant
    except Exception:
        pass
    mod = types.ModuleType("sniffles.snfp")

    @dataclass
    class PopulationVariant:                         # field set and order of snfp.py:25-37
        contig: str
        pos: int
        id: str
        alt: str
        svtype: str
        svlen: int
        end: int
        af: float
        genotyped_sample_count: int
        variant_sample_count: int

    PopulationVariant.__module__, PopulationVariant.__qualname__ = "sniffles.snfp", "PopulationVariant"
    mod.PopulationVariant = PopulationVariant
    sys.modules["sniffles.snfp"] = mod
    setattr(sys.modules["sniffles"], "snfp", mod)
    return PopulationVariant


def to_compat(call):
    """postprocess.SVCall -> the picklable candidate the reference expects (postprocessing info dropped as by SVCall.finalize)"""
    SVCall, BND, _ = compat_classes()
    names = {f.name for f in fields(SVCall)}
    kw = {k: getattr(call, k) for k in names if hasattr(call, k) and k not in ("postprocess", "bnd_info", "forward_difference_sampler")}
    b = getattr(call, "bnd_info", None)
    c = SVCall(**kw, postprocess=None, bnd_info=None if b is None else BND(b.mate_contig, b.mate_ref_start, b.is_first, b.is_reverse))
    return c


class SNFWriter:
    """one task's candidates -> a temporary part (store / annotate_block_coverages / write_and_index), then `write_results` joins the parts"""

    def __init__(self, config, handle):
        self.config, self.handle = config, handle
        self.blocks, self.index, self.total_length = {}, {}, 0

    def store(self, call):                           # snf.py:91-100
        bs = self.config.snf_block_size
        b = int(call.pos / bs) * bs
        if b not in self.blocks:
            self.blocks[b] = {t: [] for t in TYPES}
            self.blocks[b]["_COVERAGE"] = {}
        c = to_compat(call)
        if not getattr(self.config, "output_rnames", False):
            c.rnames = None
        if c.svtype in TYPES:
            self.blocks[b][c.svtype].append(c)

    def annotate_block_coverages(self, coverage_bins):
        """coverage_bins: snfb_coverage_bins(task, coverage_binsize_combine) — the reshape-mean of the contig's coverage (snf.py:248-267)"""
        step = self.config.coverage_binsize_combine
        per_block = self.config.snf_block_size // step
        for off in self.blocks:
            bi = off // self.config.snf_block_size
            for i in range(per_block):
                k = bi * per_block + i
                if -len(coverage_bins) <= k < len(coverage_bins):      # numpy indexing: a block before 0 wraps, one out of range is skipped
                    self.blocks[off]["_COVERAGE"][off + i * step] = round(float(coverage_bins[k]))

    def write_and_index(self):                       # snf.py:108-120
        offset = 0
        for b in sorted(self.blocks):
            data = gzip.compress(pickle.dumps(self.blocks[b]))
            self.handle.write(data)
            self.index[b] = (offset, len(data))
            offset += len(data)
            self.total_length += len(data)


def write_results(handle, config, parts, contigs):
    """parts: [(task_id, contig, snf_index, part_bytes, candidate_count, coverage_average_total)] -> the final .snf (snf.py:193-224)"""
    main_index, offset = {}, 0
    parts = sorted(parts, key=lambda p: p[0])
    cov = {c: [] for c in contigs}
    for task_id, contig, idx, data, n, cavg in parts:
        main_index.setdefault(contig, {})
        for block, (start, length) in idx.items():
            main_index[contig].setdefault(block, []).append((start + offset, length))
        offset += len(data)
        cov.setdefault(contig, []).append(cavg)
    cfg = dict(vars(config))
    cfg["contig_coverages"] = {c: (sum(v) / len(v) if v else 0) for c, v in cov.items()}
    header = {"config": cfg, "index": main_index, "snf_candidate_count": sum(p[4] for p in parts)}
    handle.write((json.dumps(header, default=lambda o: "<Unstored_Object>") + "\n").encode())
    for p in parts:
        handle.write(p[3])
    return header["snf_candidate_count"]


class SNFReader:
    def __init__(self, path):
        compat_classes()
        self.f = open(path, "rb")
        line = self.f.readline()
        self.header_length = len(line)
        self.header = json.loads(line.strip())
        self.index = self.header["index"]

    def close(self):
        self.f.close()

    def read_blocks(self, contig, block):            # snf.py:137-166
        ent = self.index.get(contig, {}).get(str(block))
        if ent is None:
            return None
        out = []
        for start, length in ent:
            self.f.seek(self.header_length + start)
            out.append(pickle.loads(gzip.decompress(self.f.read(length))))
        return out

    def all_calls(self):
        for contig in self.index:
            for block in sorted(self.index[contig], key=int):
                for blk in self.read_blocks(contig, block):
                    for t in TYPES:
                        for c in blk[t]:
                            yield contig, int(block), c


class PopulationReader(SNFReader):
    """a population SNF (--combine-population): an SNF whose header has a `population` record (snfp.py:110-115, 178-185) and whose blocks
    hold PopulationVariant lists.  As PopulationSNF.get_all_blocks (snf.py:235-243) only the first part of a block is read."""

    def __init__(self, path):
        super().__init__(path)
        self.population = self.header.get("population")
        self.variant_class = population_class()

    def blocks(self, contig):
        """[(block start, {svtype: [PopulationVariant, ...]})] of the contig, in index order, each block's first part"""
        out = []
        for block in self.index.get(contig, {}):
            start, length = self.index[contig][block][0]
            self.f.seek(self.header_length + start)
            out.append((int(block), pickle.loads(gzip.decompress(self.f.read(length)))))
        return out
