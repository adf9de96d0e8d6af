"""Whole-sample calling (call.call_sample) on synthetic BAMs, and the device memory of one pass.  Prints one JSON line: the card and its
power limit; per input the wall time of call_sample and its split (index and BGZF read, snfb_load_bam and snfb_run per pass, finalize,
VCF write, SNF write), the passes and their inflated bytes, at the default budget and at a budget of about 1/--passes of the BAM; and the
peak device memory of one load_bam + run over the whole BAM on a fresh context (free memory polled every millisecond).

    python scripts/call_sample_bench.py [--inputs c6,c2] [--c2-scale 0.01] [--passes 4] [--out FILE]

"c6" = bench.py --config 6's generator (four 1.5 Mb contigs, 30x, 15 kb reads); "c2" = the config-2 generator at --c2-scale.  The BAMs
(bamio.write_bam, DEFLATE level 1, noisy base qualities) go to a temporary directory."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
    name, power = [x.strip() for x in q.stdout.splitlines()[0].split(",")]
    return {"name": name, "power_limit": power}


class MemPoll:
    """the lowest free device memory seen while it runs"""

    def __enter__(self):
        import torch
        self.free, self.low, self._stop = (lambda: torch.cuda.mem_get_info(0)[0]), None, False
        self.low = self.start = self.free()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        while not self._stop:
            self.low = min(self.low, self.free())
            time.sleep(0.001)

    def __exit__(self, *exc):
        self._stop = True
        self._t.join()
        self.low = min(self.low, self.free())


def make_input(kind, scale, tmp):
    from sniffles_b200 import bamio, synth
    if kind == "c6":
        blk = synth.generate(606, [1_500_000] * 4, 30.0, len_mean=15000.0, len_sd=6000.0, sv_spacing=8000.0, phased_frac=0.3, tr_frac=0.2)
    else:
        blk = synth.config_block(2, scale)
    path = os.path.join(tmp, kind + ".bam")
    bamio.write_bam(path, blk, level=1, qual_seed=7)
    return path, len(blk.rec), int(blk.aligned_bp)


def peak_per_inflated_byte(path):
    """one snfb_load_bam + snfb_run over every contig of the BAM on a fresh context: (inflated bytes, peak device bytes)"""
    from sniffles_b200 import abi, bamio, binding, call, tasks
    from sniffles_b200 import config as sconfig
    cfg = sconfig.default_config("--all-contigs")
    bam = bamio.BamFile(path)
    planned = tasks.plan(bam.contigs, cfg)[1]
    items = list(call.task_inputs(bam, planned))
    z, spans = call.join_inputs([(it.bgzf, it.spans) for it in items])
    block = bamio.pack_records(bam.contigs, [], [(bam.name_to_id[it.contig], it.start, it.end, it.id) for it in items])
    ctx = binding.Context(0)
    ctx.set_config(abi.Config.from_sniffles(cfg))
    with MemPoll() as m:
        ctx.load_bam(z, spans, block)
        ctx.run()
    ctx.close()
    bam.close()
    return sum(it.inflated for it in items), m.start - m.low


def run_call(path, tmp, budget, tag):
    from sniffles_b200 import call
    from sniffles_b200 import config as sconfig
    vcf_path, snf_path = os.path.join(tmp, tag + ".vcf.gz"), os.path.join(tmp, tag + ".snf")
    cfg = sconfig.default_config("--input", path, "--vcf", vcf_path, "--snf", snf_path, "--all-contigs", "--allow-overwrite")
    cfg.input = path
    stats = {}
    with MemPoll() as m:
        n = call.call_sample(cfg, budget=budget, stats=stats)
    stats["peak_device_bytes_added"] = int(m.start - m.low)          # over the free memory before the call; contexts of earlier calls stay
    stats["records_written"] = n
    stats["budget"] = budget
    return stats


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--inputs", default="c6,c2")
    ap.add_argument("--c2-scale", type=float, default=0.01)
    ap.add_argument("--passes", type=int, default=4)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("call_sample_bench needs a CUDA device")
    out = {"card": card(), "device": torch.cuda.get_device_name(0), "inputs": {}}
    tmp = tempfile.mkdtemp(prefix="snfb_call_sample_")
    from sniffles_b200 import call
    for kind in a.inputs.split(","):
        t0 = time.perf_counter()
        path, n_rec, bp = make_input(kind, a.c2_scale, tmp)
        r = {"records": n_rec, "aligned_bp": bp, "bam_bytes": os.path.getsize(path), "bam_write_s": time.perf_counter() - t0}
        r["warmup"] = run_call(path, tmp, None, kind + "_warm")["wall_s"]
        infl, peak = peak_per_inflated_byte(path)
        r["one_pass_inflated_bytes"], r["one_pass_peak_device_bytes"] = infl, peak
        r["device_bytes_per_inflated_byte"] = peak / infl
        r["default_budget"] = run_call(path, tmp, None, kind + "_default")
        r["split"] = run_call(path, tmp, max(1, infl // a.passes), kind + "_split")
        r["budget_model"] = {"fixed_bytes": call.DEVICE_BYTES_FIXED, "bytes_per_inflated_byte": call.DEVICE_BYTES_PER_INFLATED_BYTE}
        out["inputs"][kind] = r
        print(f"[call_sample_bench] {kind}: {json.dumps(r)}", file=sys.stderr, flush=True)
    line = json.dumps(out)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
