"""Generates tests/golden/combine_cli/expected.json: the whole VCF the UNMODIFIED reference's combine mode writes for the cases of
tests/combine_cli_common.py, over the inputs that module derives from tests/golden/combine/sample*.snf.

The reference runs through its own code for the mode: the setup of sniffles:371-481 restated line for line below (the `sniffles` entry
forks worker processes, which the build container's stubs do not serve), its CombineTask with scatter() and execute(), its CombineResult /
CombineResultTmpFile, and its VCF writer.  The VCFs are stored in the compact form of combine_cli_common (run-stamp lines left out).
Run in the build container (needs /root/reference):
    python tests/golden/make_combine_cli_golden.py"""
import io
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, "oracle", "pyref"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import combine_cli_common as ccc                   # noqa: E402
import harness                                     # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "combine_cli")


def reference_combine_vcf(paths, extra, tmp):
    """sniffles:371-481 and 527-547 for combine mode with a plain --vcf, restated over the reference's own classes"""
    harness.import_reference()
    from sniffles import parallel, snf as refsnf, vcf as refvcf
    from sniffles.config import SnifflesConfig
    config = SnifflesConfig("--input", *paths, "--vcf", os.path.join(tmp, "out.vcf"), "--tmp-dir", tmp, *extra)
    config.mode = "combine"
    input_ext = [f.split(".")[-1].lower() for f in config.input]
    config.snf_input_info, config.sample_ids_vcf = [], []        # sniffles:156 sets the list for every mode
    pairs = []
    if len(config.input) == 1 and input_ext[0] == "tsv":
        with open(config.input[0]) as f:
            for line in f.readlines():
                s = line.strip()
                if len(s) == 0 or s[0] == "#":
                    continue
                parts = s.split("\t")
                pairs.append((parts[0], parts[1] if len(parts) == 2 else None))
    else:
        pairs = [(p, None) for p in config.input]
    for internal_id, (fn, sample_id) in enumerate(pairs):
        snf_in = refsnf.SNFile(config, open(fn, "rb"), filename=fn)
        snf_in.read_header()
        contig_lengths = snf_in.header["config"]["contig_lengths"]
        if sample_id is None:
            sample_id = snf_in.header["config"]["sample_id"] if snf_in.header["config"]["sample_id"] is not None else os.path.splitext(os.path.basename(fn))[0]
        config.snf_input_info.append({"internal_id": internal_id, "sample_id": sample_id, "filename": fn})
        snf_in.close()
    for info in config.snf_input_info:
        config.sample_ids_vcf.append((info["internal_id"], info["sample_id"]))
    if to_process := (config.contig or config.regions_by_contig):
        contig_lengths = [(name, length) for name, length in contig_lengths if name in to_process]
    result_class = None
    if len(pairs) > config.combine_max_inmemory_results:
        from sniffles.result import CombineResultTmpFile
        result_class = CombineResultTmpFile
    tasks, task_id = [], 0
    for contig_str, contig_length in contig_lengths:
        task = parallel.CombineTask(id=task_id, contig=contig_str, start=0, end=contig_length - 1, assigned_process_id=None, sv_id=0,
                                    config=config, result_class=result_class, regions=config.regions_by_contig.get(contig_str))
        tasks.extend(task.scatter())
        task_id = tasks[-1].id + 1
    buf = io.StringIO()
    vcf_out = refvcf.VCF(config, buf)
    vcf_out.write_header(contig_lengths)
    unsorted = 0
    for t in tasks:                                  # ids ascending: the order sniffles:544-547 emits finished tasks in
        t.result = t.execute()
        if result_class is not None and os.path.exists(t.result.tmpfile_unsorted):
            with open(t.result.tmpfile_unsorted) as f:
                unsorted += sum(1 for _ in f)
            os.unlink(t.result.tmpfile_unsorted)
        t.result.emit(vcf_out=vcf_out)
    lines = ccc.vcf_lines(buf.getvalue())
    return lines, [[t.id, t.contig, t.block_indices[0], t.block_indices[-1], len(t.block_indices)] for t in tasks], unsorted


def main():
    out = {"made_with": "fritzsedlazeck/Sniffles 2.8.1-dev @7fcaf867 via tests/golden/make_combine_cli_golden.py", "headers": [], "records": [],
           "cases": {}}
    pools = {"headers": {}, "records": {}}

    def index(kind, item):
        key = json.dumps(item)
        if key not in pools[kind]:
            pools[kind][key] = len(out[kind])
            out[kind].append(item)
        return pools[kind][key]
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(ccc.write_inputs(os.path.join(tmp, "in")))
        for label, files, extra in ccc.CASES:
            os.makedirs(os.path.join(tmp, label))
            lines, tasks, unsorted = reference_combine_vcf(files, extra, os.path.join(tmp, label))
            out["cases"][label] = {"inputs": files, "args": extra, "dropped": unsorted,
                                   "headers": [index("headers", x) for x in lines if isinstance(x, str)],
                                   "records": [index("records", x) for x in lines if not isinstance(x, str)],
                                   "tasks": tasks if len(tasks) <= 50 else {"n": len(tasks), "first": tasks[:3], "last": tasks[-3:]}}
            print(label, "records", sum(not isinstance(x, str) for x in lines), "tasks", len(tasks), "dropped", unsorted, flush=True)
    os.makedirs(OUT, exist_ok=True)
    with open(os.path.join(OUT, "expected.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
