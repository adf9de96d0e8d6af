"""snfb_launch_count counts the kernels the library launches, no more and no fewer: over a run, its increase equals the number of
kernel events torch.profiler records with CUDA activities (copies and memsets are not kernels)."""
import os

import pytest
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile

from sniffles_b200 import abi, bamio, binding, synth
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

BAM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bams", "hg002.bam")


@pytest.fixture(scope="module")
def ctx():
    c = binding.Context(0)
    c.set_config(abi.Config.from_sniffles(sconfig.default_config()))
    yield c
    c.close()


def _kernels_and_count(ctx, work):
    """names of the kernels the profiler saw during work(), and the increase of ctx.launch_count() over it"""
    n0 = ctx.launch_count()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        work()
    kernels = [e.name for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    return kernels, ctx.launch_count() - n0


def test_run_on_synthetic_block(ctx):
    blk = synth.generate(4242, [400_000], 20.0, len_mean=12000.0, len_sd=3000.0, sv_spacing=8000.0, tr_frac=0.2)
    ctx.load(blk)
    kernels, counted = _kernels_and_count(ctx, ctx.run)
    assert kernels, "the profiler recorded no kernel"
    assert len(kernels) == counted, sorted(set(kernels))


def test_bam_ingest_and_run(ctx):
    f = bamio.BamFile(BAM)
    bgzf, spans = f.device_input([(n, 0, L) for n, L in f.contigs])
    tables = bamio.pack_records(f.contigs, [], [(t, 0, L, t) for t, (_, L) in enumerate(f.contigs)])
    f.close()

    def work():
        ctx.load_bam(bgzf, spans, tables)
        ctx.run()
    kernels, counted = _kernels_and_count(ctx, work)
    assert any("k_inflate" in k for k in kernels), sorted(set(kernels))
    assert len(kernels) == counted, sorted(set(kernels))
