"""CPU restatement of the population lookup of combine mode (TEST INFRASTRUCTURE ONLY — never imported by sniffles_b200/).

Follows PopulationSNF.get_population_AF (/root/reference/src/sniffles/snfp.py:131-155) and PopulationVariant.match (snfp.py:91-107)
over flat arrays, in the reference's loop order: every variant of the call's (contig, block, svtype) list, in list order, is tested, and
every INS that passes the position test is aligned.  The edit distance is the Levenshtein routine of the edlib stand-in
(oracle/pyref/stubs/edlib), which the reference runs on in the golden generators.  Returns what snfb_population_match returns: the
file-order index of the best variant, -1 for none, -2 where the reference divides by a zero svlen."""
import importlib.util
import math
import os

_spec = importlib.util.spec_from_file_location("_edlib_stand_in", os.path.join(os.path.dirname(os.path.abspath(__file__)), "pyref", "stubs", "edlib", "__init__.py"))
_edlib = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_edlib)
levenshtein = _edlib.levenshtein

INS = 0


def table_lists(contig, block, svtype):
    """{(contig, block, svtype): [file-order index, ...]} of the table, list order kept; variants of contig -1 are left out"""
    out = {}
    for i, (c, b, t) in enumerate(zip(contig, block, svtype)):
        if c >= 0:
            out.setdefault((int(c), int(b), int(t)), []).append(i)
    return out


def match_one(lists, table, q, combine_match, combine_match_max, combine_pctseq, block_size):
    """table: (pos, svlen, alt) columns; q: (contig, svtype, pos, svlen, alt) of one call"""
    qc, qt, qpos, qlen, qalt = q
    if qc < 0:
        return -1
    pos, svlen, alt = table
    best_dist, best = None, -1
    for i in lists.get((int(qc), int(int(qpos / block_size) * block_size), int(qt)), []):
        dist = abs(int(pos[i]) - qpos) + abs(abs(int(svlen[i])) - abs(qlen))
        minlen = float(min(abs(int(svlen[i])), abs(qlen)))
        if dist > combine_match * math.sqrt(minlen) or dist > combine_match_max:
            continue
        if qt == INS and combine_pctseq:
            d = levenshtein(alt[i], qalt)
            if int(svlen[i]) == 0:
                return -2
            if (int(svlen[i]) - d) / int(svlen[i]) <= combine_pctseq:
                continue
        if best_dist is None or dist < best_dist:
            best_dist, best = dist, i
    return best


def match(table, queries, combine_match, combine_match_max, combine_pctseq, block_size):
    """table: dict of contig, block, svtype, pos, svlen, alt (file order); queries: dict of contig, svtype, pos, svlen, alt -> [best]"""
    lists = table_lists(table["contig"], table["block"], table["svtype"])
    cols = (table["pos"], table["svlen"], table["alt"])
    return [match_one(lists, cols, (int(c), int(t), int(p), int(s), a), combine_match, combine_match_max, combine_pctseq, block_size)
            for c, t, p, s, a in zip(queries["contig"], queries["svtype"], queries["pos"], queries["svlen"], queries["alt"])]
