"""Combine mode end to end on the GPU: a seeded config-4-shaped cohort (bench.combine_workload: 50 samples sharing planted sites on 24
GRCh38-length contigs, scaled) written as SNF files, then combine_run.combine_snfs over them.  Prints one JSON line: the wall time and
its split from `stats` (headers, SNF block decode, device, call_group, VCF write), the device intervals of the plan and the grouping from
snfb_last_timings of the last pass, and a CPU arm: CombineTask.plan + plan_arrays over the tasks of the first pass.

    python scripts/combine_sample_bench.py [--scale 0.1] [--out DIR]"""
import argparse
import gzip
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def write_cohort(directory, scale, n_samples=50):
    """bench.combine_workload's candidates as one SNF per sample (header + gzip(pickle) blocks, as snf.SNFWriter lays them out)"""
    import bench
    from sniffles_b200 import snf
    SVCall, BND, _ = snf.compat_classes()
    lens, readers = bench.combine_workload(n_samples, scale)
    contigs = [(f"ctg{i + 1}", n) for i, n in enumerate(lens)]
    paths = []
    for k, rd in enumerate(readers):
        index, parts, off, count = {}, [], 0, 0
        for (contig, b), blk in sorted(rd.d.items(), key=lambda kv: ([c for c, _ in contigs].index(kv[0][0]), kv[0][1])):
            out = {"_COVERAGE": blk["_COVERAGE"]}
            for t in snf.TYPES:
                out[t] = []
                for c in blk[t]:
                    end = c.pos + abs(c.svlen)
                    s = SVCall(contig=contig, pos=c.pos, id=f"{t}.{count:X}", ref="N", alt=c.alt, qual=30, filter="PASS", info={}, svtype=t, svlen=c.svlen,
                               end=end, genotypes={0: (0, 1, 30, 20, c.support, (None, None))}, precise=True, support=c.support, rnames=None, qc=True,
                               nm=-1, postprocess=None, fwd=1, rev=1, coverage_upstream=30, coverage_downstream=30, coverage_start=30, coverage_center=30,
                               coverage_end=30)
                    if c.bnd_info is not None:
                        s.bnd_info = BND(c.bnd_info.mate_contig, c.bnd_info.mate_ref_start, True, False)
                    out[t].append(s)
                    count += 1
            data = gzip.compress(pickle.dumps(out))
            index.setdefault(contig, {})[b] = [(off, len(data))]
            parts.append(data)
            off += len(data)
        header = {"config": {"snf_block_size": 100000, "snf_format_version": "S2_rc4", "sample_id": f"S{k}", "build": "2.8.1",
                             "contig_lengths": contigs}, "index": index, "snf_candidate_count": count}
        p = os.path.join(directory, f"s{k}.snf")
        with open(p, "wb") as f:
            f.write((json.dumps(header) + "\n").encode())
            for data in parts:
                f.write(data)
        paths.append(p)
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=0.1)
    ap.add_argument("--out", default=None, help="directory for the VCF (default: a temporary one)")
    args = ap.parse_args()
    import torch
    from sniffles_b200 import combine, combine_run, snf, tasks
    from sniffles_b200 import config as sconfig
    if not torch.cuda.is_available():
        raise SystemExit("combine_sample_bench needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    with tempfile.TemporaryDirectory() as tmp:
        t0 = time.perf_counter()
        paths = write_cohort(tmp, args.scale)
        write_s = time.perf_counter() - t0
        out_dir = args.out or tmp
        os.makedirs(out_dir, exist_ok=True)
        vcf_path = os.path.join(out_dir, "combined.vcf")
        cfg = sconfig.SnifflesConfig("-i", *paths, "-v", vcf_path, "--allow-overwrite")
        tasks.device_context(0)                                      # context creation outside the timed run
        st = {}
        n = combine_run.combine_snfs(cfg, stats=st)
        timings = tasks.device_context(0).timings()
        # CPU arm: the host restatement of the plan (SNF decode included) over the tasks of the first pass
        planned = combine_run.plan_tasks(cfg, combine_run.read_inputs(cfg)[0])
        first = planned[:st["pass_tasks"][0]]
        readers = {s["internal_id"]: snf.SNFReader(s["filename"]) for s in cfg.snf_input_info}
        t1 = time.perf_counter()
        plan = combine.Plan()
        for k, t in enumerate(first):
            t.plan(readers, plan, k)
        combine.plan_arrays(plan, cfg)
        cpu_plan_s = time.perf_counter() - t1
        for r in readers.values():
            r.close()
    dev = {name: round(ms, 3) for name, ms, _ in timings}
    print(json.dumps({"workload": f"config-4 shape: 50 samples, scale {args.scale}", "gpu": gpu, "records": n, "passes": st["passes"],
                      "candidates": sum(st["pass_candidates"]), "wall_s": round(st["wall_s"], 3), "header_s": round(st["header_s"], 3),
                      "decode_s": round(st["decode_s"], 3), "device_s": round(st["device_s"], 3), "call_group_s": round(st["call_group_s"], 3),
                      "write_s": round(st["write_s"], 3), "dropped": st["dropped"], "device_ms_last_pass": dev,
                      "cpu_plan_s_incl_decode": round(cpu_plan_s, 3), "snf_write_s": round(write_s, 3)}))


if __name__ == "__main__":
    main()
