"""developer aid: where does consensus::k_align spend its time?  (run with SNFB_DEBUG=1)"""
import ctypes as C, os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["SNFB_DEBUG"] = "1"
import __graft_entry__ as g; g.build()
from sniffles_b200 import abi, binding, synth, config as sconfig
scale = float(sys.argv[1]) if len(sys.argv) > 1 else 0.25
cfgi = int(sys.argv[2]) if len(sys.argv) > 2 else 2
blk = synth.config_block(cfgi, scale)
ctx = binding.Context(0); ctx.set_config(abi.Config.from_sniffles(sconfig.default_config())); ctx.load(blk)
for _ in range(3): res = ctx.run(want_leads=False)
print({n: round(ms, 3) for n, ms, _ in ctx.timings()})
nw = 132 * 7 * 4          # k_align grid (NUM_SMS * 7) x ALIGN_WARPS
out = np.zeros(nw * 8, "<u8")
rc = binding.lib().snfb_debug_dump(ctx._h, out.ctypes.data, len(out)); print("rc", rc)
d = out.reshape(nw, 8)
busy, total, items = (d[:, i].astype(np.float64) for i in range(3))
ph = d[:, 3:8].astype(np.float64).sum(axis=0)
print("warps", nw, "items", int(items.sum()), "cands", len(res.cand))
print("elapsed cycles per warp: min %.0f median %.0f max %.0f" % (total.min(), np.median(total), total.max()))
print("busy  cycles per warp: median %.0f max %.0f" % (np.median(busy), busy.max()))
print("cycles per item: mean %.0f" % (busy.sum() / max(items.sum(), 1)))
names = ["unpack", "probe", "automaton+segments(3a)", "run filter(3b)", "row write(3c)"]
print("phase shares:", {n: round(float(v / ph.sum()), 3) for n, v in zip(names, ph)})
