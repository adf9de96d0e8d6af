"""Generates tests/golden/reference/snf_coverage.json: the `_COVERAGE` entries of every SNF block the UNMODIFIED reference writes with
`--snf` and `--reference` (oracle/pyref/harness.py behind its stub pysam) for the golden FASTA blocks of tests/ref_fasta.py.  Runs only
where the reference tree exists; the fixture travels, the reference does not.

    python tests/golden/make_snf_coverage_golden.py

The reference masks its per-base coverage vector with the FASTA's 'N' runs (LeadProvider._mask_N_coverage, leadprov.py:470) before
SNFile.annotate_block_coverages averages it (snf.py:249-267), so these bins pin the masked means.  The same block is written once more
without --reference and at least one stored value must differ, or the fixture would not pin the mask at all."""
import json
import logging
import os
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle", "pyref"), os.path.join(ROOT, "tests"), HERE]
logging.disable(logging.CRITICAL)

import harness  # noqa: E402
import ref_fasta  # noqa: E402
from make_golden import FIXTURES  # noqa: E402
from make_reference_golden import TextFasta  # noqa: E402
from sniffles_b200 import snf, synth  # noqa: E402


def coverage_of(path):
    """{contig: {block offset: {position: mean}}} of every block of an SNF file"""
    rd = snf.SNFReader(path)
    out = {}
    for contig, blocks in rd.index.items():
        for off in sorted(blocks, key=int):
            (b,) = rd.read_blocks(contig, off)
            out.setdefault(contig, {})[str(off)] = {str(k): int(v) for k, v in sorted(b["_COVERAGE"].items())}
    rd.close()
    return out


def main():
    harness.import_reference()
    import pysam
    pysam.FastaFile = TextFasta
    out = dict(made_with="fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via oracle/pyref/harness.py", blocks={})
    tmp = tempfile.mkdtemp()
    n_diff = 0
    for name in ref_fasta.GOLDEN_FASTA:
        text, _ = ref_fasta.golden_fasta(name)
        fa = os.path.join(tmp, name + ".fa")
        with open(fa, "wb") as f:
            f.write(text)
        kw, args = FIXTURES[name]
        kw2 = dict(kw)
        blk = synth.generate(kw2.pop("seed"), kw2.pop("contig_len"), kw2.pop("coverage"), **kw2)
        masked = coverage_of(harness.write_reference_snf(blk, args, os.path.join(tmp, name + ".masked.snf"), reference=fa))
        plain = coverage_of(harness.write_reference_snf(blk, args, os.path.join(tmp, name + ".plain.snf")))
        assert masked.keys() == plain.keys() and all(masked[c].keys() == plain[c].keys() for c in masked)
        diff = sum(masked[c][b][p] != plain[c][b][p] for c in masked for b in masked[c] for p in masked[c][b])
        n_diff += diff
        out["blocks"][name] = dict(fasta_sha256=ref_fasta.sha256(text), args=args, coverage=masked)
        print(name, "blocks", sum(len(v) for v in masked.values()), "bins moved by the mask", diff, flush=True)
    assert n_diff > 0, "no stored _COVERAGE value differs from the unmasked one: the fixture would not pin the mask"
    with open(os.path.join(HERE, "reference", "snf_coverage.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
