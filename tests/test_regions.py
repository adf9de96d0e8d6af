"""`--regions` / `--region` without a GPU: the parser against the reference's own parsing (tests/golden/regions/expected.json), the
--contig conflict, the fetch windows pysam would refuse, the region table and span tags, and the N runs clipped to the regions."""
import json
import logging
from unittest.mock import mock_open, patch

import numpy as np
import pytest

import regions_common as rc
from sniffles_b200 import abi, call, fasta, tasks
from sniffles_b200 import config as sconfig

with open(rc.EXPECTED) as _f:
    EXPECTED = json.load(_f)


def _flat(cfg):
    return {c: [list(r) for r in v] for c, v in cfg.regions_by_contig.items()}


@pytest.mark.parametrize("key", ["good_file", "invalid_lines", "unsorted_overlap"])
def test_bed_parsing_matches_reference(key):
    want = EXPECTED["parser"][key]
    with patch("builtins.open", mock_open(read_data=want["bed"])):
        cfg = sconfig.SnifflesConfig("--input", "input.bam", "--vcf", "out.vcf", "--regions", "regions.bed")
    assert _flat(cfg) == want["regions_by_contig"]


def test_region_strings_match_reference(caplog):
    want = EXPECTED["parser"]["region_strings"]
    with caplog.at_level(logging.WARNING):
        cfg = sconfig.SnifflesConfig("--input", "input.bam", "--vcf", "out.vcf", *[x for s in want["strings"] for x in ("--region", s)])
    assert _flat(cfg) == want["regions_by_contig"]
    assert "skipping region 'bad'" in caplog.text


def test_regions_file_wins_over_region_strings(tmp_path):
    bed = tmp_path / "r.bed"
    bed.write_text("chr9\t1\t2\n")
    cfg = sconfig.SnifflesConfig("--input", "i.bam", "--vcf", "o.vcf", "--regions", str(bed), "--region", "chr1:5-9")
    assert _flat(cfg) == {"chr9": [["chr9", 1, 2]]}


def test_contig_and_regions_conflict():
    with pytest.raises(SystemExit):
        sconfig.SnifflesConfig("--input", "i.bam", "--vcf", "o.vcf", "--regions", "regions.bed", "-c", "chr6")


def test_missing_regions_file():
    with pytest.raises(FileNotFoundError):
        sconfig.SnifflesConfig("--input", "i.bam", "--vcf", "o.vcf", "--regions", "/nonexistent/regions.bed")


def test_regions_select_contigs():
    cfg = sconfig.SnifflesConfig("--input", "i.bam", "--vcf", "o.vcf", "--region", "short:0-10")
    processed, planned = tasks.plan([("long", 5_000_000), ("short", 1000)], cfg)
    assert processed == [("short", 1000)] and planned == [(0, "short", 0, 999)]


def test_fetch_windows():
    def R(c, s, e):
        return (c, s, e)
    assert tasks.fetch_windows("c", 0, 99, None) == [(0, 99)]
    assert tasks.fetch_windows("c", 0, 99, [R("c", 50, 60), R("c", 10, 70), R("c", 5, 5)]) == [(50, 60), (10, 70), (5, 5)]
    with pytest.raises(ValueError):
        tasks.fetch_windows("c", 0, 99, [R("c", 10, 20), R("c", 30, 29)])
    with pytest.raises(ValueError):
        tasks.fetch_windows("c", 0, 99, [R("c", -1, 20)])
    t = tasks.region_table([(0, [(5, 9), (1, 3)]), (1, [(0, 99)])])
    assert t.dtype == abi.REGION_DTYPE and t.tolist() == [(0, 5, 9, 0), (0, 1, 3, 0), (1, 0, 99, 0)]


def test_join_inputs_rebases_region_tags():
    sp = np.zeros(2, abi.SPAN_DTYPE)
    sp["region"] = [0, 1]
    _, spans = call.join_inputs([(np.zeros(4, "u1"), sp), (np.zeros(4, "u1"), sp[:1].copy())], [2, 3])
    assert spans["task"].tolist() == [0, 0, 1] and spans["region"].tolist() == [0, 1, 2]
    assert spans["cbeg"].tolist() == [0, 0, 4]


def _ref(length, runs):
    r = object.__new__(fasta.Reference)
    r._row, r._slot, r._runs = {"c": {"length": length}}, {"c": 0}, {"c": np.asarray(runs, np.int32).reshape(-1, 2)}
    return r


def test_n_runs_clipped_to_regions():
    ref = _ref(1000, [(0, 10), (95, 130), (400, 500), (990, 1000)])
    # out of order, overlapping and adjacent regions; the mask is zero outside them
    got = ref.region_runs("c", [(100, 200), (450, 460), (120, 300), (300, 420), (995, 2000)], 1000)
    assert got.tolist() == [[100, 130], [400, 420], [450, 460], [995, 1000]]


def test_one_region_the_fasta_cannot_serve_voids_the_mask(caplog):
    ref = _ref(800, [(0, 10)])                      # FASTA contig shorter than the BAM's 1000
    with caplog.at_level(logging.WARNING):
        assert ref.region_runs("c", [(0, 100), (700, 900)], 1000) is None
    assert "Unable to mask N regions" in caplog.text
    assert ref.region_runs("c", [(0, 100), (700, 790)], 1000).tolist() == [[0, 10]]
    assert ref.region_runs("missing", [(0, 100)], 1000) is None
    # a single fetched base broadcast over its slice: all N or nothing
    assert _ref(6, []).region_runs("c", [(5, 900)], 806).tolist() == []
    assert _ref(6, [(5, 6)]).region_runs("c", [(5, 900)], 806).tolist() == [[5, 806]]


def test_device_input_tags_regions_and_ships_shared_blocks_once(tmp_path):
    import call_sample_common as csc
    from sniffles_b200 import bamio
    paths = csc.write_inputs("c1_ont_1mb", str(tmp_path))
    bam = bamio.BamFile(paths["bam"])
    (name, L), = rc.contigs_with_reads(bam)[:1]
    one_z, one = bam.device_input([(name, L // 4, L // 2)])
    z, spans = bam.device_input([(name, L // 4, L // 2), (name, L // 4, L // 2), (name, L // 3, L // 2)], tags=[(0, 0), (0, 1), (0, 2)])
    assert np.array_equal(z, one_z)                  # the same blocks, once, for three overlapping queries
    assert spans["task"].tolist() == [0] * len(spans)
    assert (spans["region"] == 0).sum() == (spans["region"] == 1).sum() == len(one) and (spans["region"] == 2).sum() > 0
    assert np.array_equal(spans[spans["region"] == 1][["cbeg", "cend", "ubeg", "uend"]], one[["cbeg", "cend", "ubeg", "uend"]])
    bam.close()
