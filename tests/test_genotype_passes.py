"""genotype.genotype_vcf's handling of a device pass the library refuses, without a GPU: a stand-in context whose snfb_load_bam fails
makes the run raise call.CallSampleError naming the pass's contigs and inflated bytes, and the command line exit with the fatal-error
line and code 1, no traceback."""
import pytest

import call_sample_common as csc
import test_genotype_parity as tgp
from sniffles_b200 import __main__ as cli
from sniffles_b200 import binding, call, genotype, tasks


class RefusingContext:
    """takes a pass's configuration and regions, refuses its load as snfb_load_bam refuses one"""

    def set_config(self, cfg):
        pass

    def set_regions(self, table):
        pass

    def load_bam(self, bgzf, spans, block):
        raise binding.SnfbError("snfb_load_bam: out of device memory")

    def run(self, **kw):
        raise AssertionError("run after a refused load")


@pytest.fixture
def refusing(monkeypatch):
    monkeypatch.setattr(tasks, "device_context", lambda device=0: RefusingContext())
    monkeypatch.setattr(call, "device_budget", lambda device=0: 1 << 40)


@pytest.fixture
def phased(tmp_path):
    fx, _ = tgp.load("phased_phase")
    return fx, csc.write_inputs("phased_phase", str(tmp_path / "in"))


def test_refused_pass_raises_call_sample_error(refusing, phased, tmp_path):
    fx, paths = phased
    for budget, named in ((1 << 40, "ctg1, ctg2"), (1, "ctg1")):
        cfg = tgp.config_for(fx, "--input", paths["bam"], "--vcf", str(tmp_path / "out.vcf"))
        cfg.input = paths["bam"]
        stats = {}
        with pytest.raises(call.CallSampleError, match=rf"contig\(s\) {named} \(\d+ inflated BAM bytes\) failed: snfb_load_bam: out of device memory"):
            genotype.genotype_vcf(cfg, budget=budget, stats=stats)
        assert stats["passes"] == 0


def test_command_line_exits_with_the_fatal_error(refusing, phased, tmp_path, caplog, capsys):
    fx, paths = phased
    args = ["--input", paths["bam"], "--vcf", str(tmp_path / "out.vcf"), "--genotype-vcf", tgp.config_for(fx).genotype_vcf, *fx["args"]]
    assert cli.main(args) == 1
    err = [r for r in caplog.records if r.levelname == "ERROR"]
    assert len(err) == 1 and err[0].getMessage().endswith("out of device memory (Fatal error, exiting.)")
    assert "contig(s) ctg1, ctg2" in err[0].getMessage() and err[0].exc_info is None
    captured = capsys.readouterr()
    assert "Traceback" not in captured.out + captured.err + caplog.text
