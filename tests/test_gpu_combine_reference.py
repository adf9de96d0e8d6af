"""Combine mode with `--reference` on the device against the reference's combine mode (tests/golden/combine_reference, made by
tests/golden/make_combine_reference_golden.py over the inputs of combine_cli_common and the seeded FASTA of combine_reference_common):
the whole VCF for every case, .vcf.gz output, the output at a pass budget of one task, a BGZF FASTA, and the runs without a usable FASTA
against tests/golden/combine_cli."""
import gzip
import logging
import os

import pytest

import combine_cli_common as ccc
import combine_reference_common as crc
from sniffles_b200 import __main__ as cli, bamio, combine_run
from sniffles_b200 import config as sconfig

pytestmark = pytest.mark.gpu

SHA, GOLD = crc.load_expected()
CLI_GOLD = ccc.load_expected()
CASES = {label: (files, extra, kind, population) for label, files, extra, kind, population in crc.CASES}


@pytest.fixture(scope="module")
def inputs(tmp_path_factory):
    """(SNF input directory, {FASTA kind: path}); the FASTAs are the golden data's"""
    d = tmp_path_factory.mktemp("combine_reference")
    fastas = {}
    for kind in ("full", "no_ctg2"):
        fastas[kind], sha = crc.fasta_files(kind, str(d))
        assert sha == SHA[kind], kind
    return ccc.write_inputs(str(d / "in")), fastas


def _args(label, fastas, out):
    files, extra, kind, population = CASES[label]
    return crc.case_args(files, extra, population, out, fastas[kind])


def _lines(path):
    data = open(path, "rb").read()
    return ccc.vcf_lines((gzip.decompress(data) if path.endswith(".gz") else data).decode())


def test_cases_are_the_golden_ones():
    assert sorted(GOLD) == sorted(CASES)
    for label, case in GOLD.items():
        files, extra, kind, population = CASES[label]
        assert [case["inputs"], case["args"], case["fasta"], case["population"]] == [files, extra, kind, population]
    # the golden runs meet the allele rules: DEL REF bases, anchored INS / BND, DELs dropped for their N, a contig left out
    assert GOLD["in_memory"]["alleles"]["del_sequence"] > 0 and GOLD["in_memory"]["alleles"]["anchored"] > 0
    assert len(GOLD["max_unknown"]["records"]) < len(GOLD["in_memory"]["records"]) < len(GOLD["symbolic"]["records"])
    assert GOLD["contig_absent"]["alleles"]["n_ref"] > GOLD["in_memory"]["alleles"]["n_ref"]


@pytest.mark.parametrize("label", sorted(CASES))
def test_command_line_matches_the_reference(label, inputs, tmp_path, monkeypatch, caplog):
    d, fastas = inputs
    monkeypatch.chdir(d)
    out = str(tmp_path / "out.vcf")
    caplog.set_level(logging.INFO)
    assert cli.main(_args(label, fastas, out)) == 0
    assert _lines(out) == GOLD[label]["vcf"]
    assert crc.allele_counts(open(out).read()) == GOLD[label]["alleles"]
    assert f"Opening for reading: {fastas[CASES[label][2]]}" in caplog.text


@pytest.mark.parametrize("label", ["in_memory", "population", "contig_absent"])
def test_compressed_output(label, inputs, tmp_path, monkeypatch):
    d, fastas = inputs
    monkeypatch.chdir(d)
    gz = str(tmp_path / "out.vcf.gz")
    assert cli.main(_args(label, fastas, gz)) == 0
    assert _lines(gz) == GOLD[label]["vcf"] and os.path.getsize(gz + ".tbi") > 0


@pytest.mark.parametrize("label", ["in_memory", "tmpfile", "regions", "population"])
def test_pass_budgets_give_the_same_file(label, inputs, tmp_path, monkeypatch):
    d, fastas = inputs
    monkeypatch.chdir(d)
    texts = []
    for budget in (1, None):
        out = str(tmp_path / f"b{budget}.vcf")
        st = {}
        combine_run.combine_snfs(sconfig.SnifflesConfig(*_args(label, fastas, out)), budget=budget, stats=st)
        assert st["dropped"] == GOLD[label]["dropped"]
        assert len(st["prefetch_s"]) == len(st["prefetch_bytes"]) == st["passes"]          # bases cached by an earlier run are not gathered again
        if budget == 1:
            assert st["passes"] >= 2
        texts.append(_lines(out))
    assert texts[0] == texts[1] == GOLD[label]["vcf"]


def _bgzf(path, fai, out=None):
    text = open(path, "rb").read()
    out = out or path + ".gz"
    with open(out, "wb") as f:
        for k in range(0, len(text), 0xff00):
            f.write(bamio._bgzf_block(text[k:k + 0xff00]))
        f.write(bamio._BGZF_EOF)
    if fai:
        with open(out + ".fai", "wb") as f:
            f.write(open(path + ".fai", "rb").read())
    return out


def test_bgzf_fasta(inputs, tmp_path, monkeypatch):
    d, fastas = inputs
    monkeypatch.chdir(d)
    out = str(tmp_path / "out.vcf")
    args = _args("in_memory", fastas, out)
    args[args.index("--reference") + 1] = _bgzf(fastas["full"], fai=True)
    assert cli.main(args) == 0
    assert _lines(out) == GOLD["in_memory"]["vcf"]


def test_without_a_usable_fasta_the_output_is_the_combine_golden(inputs, tmp_path, monkeypatch, caplog):
    """no --reference, a BGZF FASTA without its .fai, a stale .fai: the records of tests/golden/combine_cli"""
    d, fastas = inputs
    monkeypatch.chdir(d)
    for label in ("default4", "tmpfile"):
        bgzf = _bgzf(fastas["full"], fai=False, out=str(tmp_path / f"{label}.fa.gz"))
        stale = str(tmp_path / f"{label}_stale.fa")
        with open(stale, "wb") as f:
            f.write(open(fastas["full"], "rb").read())
        fai = open(fastas["full"] + ".fai").read().splitlines()
        fai[0] = fai[0].replace("\t60\t61", "\t61\t62")          # ctg1 written at 60 columns, indexed as 61
        with open(stale + ".fai", "w") as f:
            f.write("\n".join(fai) + "\n")
        case = CLI_GOLD[label]
        for k, extra in enumerate(([], ["--reference", bgzf], ["--reference", stale])):
            out = str(tmp_path / f"{label}{k}.vcf")
            caplog.clear()
            assert cli.main(["-i", *case["inputs"], "-v", out, *case["args"], *extra]) == 0
            assert _lines(out) == case["vcf"], (label, extra)
            errors = [r.getMessage() for r in caplog.records if r.levelno >= logging.ERROR]
            assert len(errors) == (1 if extra else 0) and all("Unable to open reference file" in e for e in errors), errors
