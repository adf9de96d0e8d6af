"""Force calling against the unmodified reference's GenotypeTask.execute (tests/golden/genotype/<block>.expected.json, written by
make_genotype_golden.py): the C oracle's candidates, the plain-Python restatement of the matching and target coverage
(oracle/genotype.py) and the host epilogue and writer reproduce every output line, the header included, and drop the same tasks.
The GPU variant (test_gpu_genotype.py) runs the same fixtures through a BAM and the device."""
import io
import json
import os

import pytest

import oracle.oracle as orc
from oracle import genotype as ogt
from sniffles_b200 import abi, genotype, tasks
from sniffles_b200 import config as sconfig

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "genotype")
BLOCKS = ["c1_ont_1mb", "phased_phase", "c3_hifi_mosaic", "hg008"]


def load(name):
    import test_oracle_golden as tog
    with open(os.path.join(G, name + ".expected.json")) as f:
        fx = json.load(f)
    blk = tog._bam_block("hg008") if name == "hg008" else tog.load_fixture(name)[1]
    return fx, blk


def config_for(fx, *extra):
    cfg = sconfig.default_config(*fx["args"], "--genotype-vcf", os.path.join(G, fx["block"] + ".targets.vcf"), *extra)
    for k, v in fx["stamp"].items():
        setattr(cfg, k, v)
    return cfg


@pytest.mark.parametrize("name", BLOCKS)
def test_oracle_and_epilogue_reproduce_reference(name):
    from test_gpu_full_size import numpy_filter
    fx, blk = load(name)
    cfg = config_for(fx)
    header, targets = genotype.read_targets(cfg.genotype_vcf)
    contigs = [(n, int(c["length"])) for n, c in zip(blk.contig_names, blk.contig)]
    task_of = {blk.contig_names[int(blk.task[t]["contig"])]: t for t in range(len(blk.task))}
    jobs = [p + (task_of[p[1]],) for p in genotype.plan(contigs, targets, cfg) if p[4]]
    res = orc.run(blk, abi.Config.from_sniffles(cfg), 3, 2, keep_rec_nm=True)
    br = tasks.BlockRun(blk, res, tasks.cand_ranges(res.cand, len(blk.task)), res.rec_nm)
    ok, _ = numpy_filter(blk, cfg)
    span = ogt.record_spans(blk)
    br.genotype = {}
    for _, _, _, _, ts, k in jobs:
        lo, hi = br.cand_range[k]
        br.genotype[k] = ogt.task_results(ogt.cand_svs(res.cand[lo:hi], blk.contig_names), lo, ts, ogt.coverage_vector(blk, ok, span, k),
                                          cfg.combine_match, cfg.combine_match_max, cfg.cluster_merge_bnd, cfg.coverage_binsize)
    out = io.StringIO()
    out.write(genotype.rewrite_header(header, cfg))
    n = genotype.write_tasks(out, br, jobs, cfg)
    assert n == fx["n_written"]
    assert out.getvalue() == fx["output"]
