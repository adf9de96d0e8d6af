"""Generates tests/golden/reference/golden.json from the UNMODIFIED reference run with `--reference` (oracle/pyref/harness.py behind
its stub pysam), for the c2_ont_wgs_small and phased_phase blocks and the seeded FASTAs of tests/ref_fasta.py.  Runs only where the
reference tree exists; the fixture travels, the reference does not.

    python tests/golden/make_reference_golden.py

The stub `pysam.FastaFile` is replaced by a reader of the real FASTA text (test infrastructure, here only), so the reference's own
LeadProvider._mask_N_coverage and VCF.write_call read it.  Stored per block: the fields of the candidates as they leave
Task.call_candidates that the N mask can move (the coverage probes; the same for every argument set) and the contig mean coverage; per
argument set the VCF lines VCF.write_call emits for the finalized calls, as ref_fasta.vcf_digest stores them."""
import json
import logging
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests")]
logging.disable(logging.CRITICAL)

import harness  # noqa: E402
import ref_fasta  # noqa: E402
from make_golden import FIXTURES  # noqa: E402
from sniffles_b200 import synth  # noqa: E402

ARGSETS = {"default": [], "symbolic": ["--symbolic"], "short_del_seq": ["--max-del-seq-len", "100", "--max-unknown-pct", "0.1"]}


class TextFasta:
    """pysam.FastaFile over a FASTA text: fetch as pysam resolves it (KeyError for an unknown name, ValueError for start < 0 or
    start > end, end clipped to the length)"""

    def __init__(self, path):
        self.seqs, name = {}, None
        with open(path) as f:
            for line in f:
                line = line.rstrip("\r\n")
                if line.startswith(">"):
                    name = line[1:].split()[0]
                    self.seqs[name] = []
                else:
                    self.seqs[name].append(line)
        self.seqs = {k: "".join(v) for k, v in self.seqs.items()}

    def fetch(self, contig, start=None, end=None):
        s = self.seqs[contig]
        start = 0 if start is None else start
        end = len(s) if end is None else end
        if start < 0 or start > end:
            raise ValueError("invalid coordinates")
        return s[start:min(end, len(s))]


def main():
    harness.import_reference()
    import pysam
    pysam.FastaFile = TextFasta
    out = dict(made_with="fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", blocks={})
    tmp = tempfile.mkdtemp()
    for name in ref_fasta.GOLDEN_FASTA:
        text, _ = ref_fasta.golden_fasta(name)
        path = os.path.join(tmp, name + ".fa")
        with open(path, "wb") as f:
            f.write(text)
        kw, base_args = FIXTURES[name]
        kw2 = dict(kw)
        blk = synth.generate(kw2.pop("seed"), kw2.pop("contig_len"), kw2.pop("coverage"), **kw2)
        entry = dict(fasta_sha256=ref_fasta.sha256(text), tasks=None, args={})
        for key, extra in ARGSETS.items():
            cfg = harness.make_config(*base_args, *extra)
            cfg.reference = path
            harness.FakeFasta = lambda: TextFasta(path)         # the writer's handle (run_task's "vcf_ref" lines)
            tasks, vcf = [], []
            for t in range(len(blk.task)):
                r = harness.run_task(blk, t, cfg)
                tasks.append(dict(cands=[[c[k] for k in ref_fasta.CAND_FIELDS] for c in r["cands"]], cov_mean=r["cov_mean"], read_count=r["read_count"]))
                vcf.append([ref_fasta.vcf_digest(line) for line in r["vcf_ref"]])
            assert entry["tasks"] in (None, tasks), "the candidates differ between argument sets"
            entry["tasks"] = tasks
            entry["args"][key] = dict(argv=base_args + extra, vcf=vcf)
            print(name, key, "cands", sum(len(t["cands"]) for t in tasks), "vcf lines", sum(len(v) for v in vcf), flush=True)
        out["blocks"][name] = entry
    os.makedirs(os.path.join(HERE, "reference"), exist_ok=True)
    with open(os.path.join(HERE, "reference", "golden.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
