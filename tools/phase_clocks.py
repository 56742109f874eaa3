"""Per-phase cycle attribution of sparse_img_align_kernel at the bench.py workload (B = 1024 VGA pairs, 300 points +
80 segments, levels 4 -> 2, seed 3000, <128,4>).

Needs a library built with the opt-in clocks, selected with PLSVO_LIB:
    python -c "import sys; sys.path.insert(0, 'pl-svo_b200'); import build; build.build_variant('phase', ['PLSVO_PHASE_CLOCKS'])"
    PLSVO_LIB=pl-svo_b200/csrc/libplsvo_b200_phase.so python tools/phase_clocks.py
Every warp's lane 0 adds the clock64() cycles between its marks to the phase they close, so a share is a share of
warp-resident time.  The clock reads cost a little themselves: use the shares, not the absolute rate.

The serial section of a pass is reported by sub-phase twice: as warp cycles per pass (over the CTA's warps, so the
sub-phases add up to the serial section of the pass table) and as cycles per pass summed over the warps that run the
sub-phase.  The cross-warp sum, the solve and the decision run on warp 0, the walk on warp 1 and the segment sum on
warp 2, so for those the second figure is their latency in a pass.  Two sub-phases are sums over several warps: the
barrier waits (three warps at named barrier 1, all four at the final block barrier), and the decision, whose mark every
warp passes, so warps 1-3 add the short gap since their previous mark to thread 0's decision time."""
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "oracle")]
import numpy as np
import torch

import plsvo_b200
from plsvo_b200 import abi, synth

SERIAL = ["cross_warp_sum", "solve", "walker", "segment_sum", "named_barrier_1", "decide", "final_barrier"]
PHASES = ["setup_precompute", "point_eval", "point_chi2_barrier", "segment_rounds", "block_reduce"] + SERIAL + ["pair_other"]
PASS = slice(1, 1 + 4 + len(SERIAL))   # point_eval .. final_barrier
SER = slice(5, 5 + len(SERIAL))

steps = int(os.environ.get("PHASE_STEPS", 5))
dev = torch.device("cuda", 0)
data = synth.make_align_batch(batch=1024, n_pts=300, n_segs=80, device=dev, seed=3000)
stream = torch.cuda.Stream(dev)
torch.cuda.set_stream(stream)
ctx = plsvo_b200.Context(0, stream.cuda_stream)
al = plsvo_b200.SparseImgAlign(4, 2, 30, ctx=ctx)
lib = abi.load_library()
read = lib.plsvo_phase_clocks  # AttributeError: PLSVO_LIB is not a -DPLSVO_PHASE_CLOCKS build
read.restype, read.argtypes = C.c_int, [C.POINTER(C.c_ulonglong), C.c_int]
buf = (C.c_ulonglong * len(PHASES))()

al.upload(data)
al.launch()
ctx.sync()
assert read(buf, 1) == 0
for _ in range(steps):
    al.launch()
ctx.sync()
assert read(buf, 1) == 0
out = al.download()
cyc = np.array(buf[:], dtype=np.float64)
passes = steps * int(out.iters.sum())
warps = 128 // 32
pass_total = cyc[PASS].sum()
per_pass = {
    "point_eval": cyc[1], "point_chi2_barrier": cyc[2], "segment_rounds": cyc[3], "block_reduce": cyc[4],
    "serial": cyc[SER].sum(),
}
print(json.dumps({
    "lib": os.environ.get("PLSVO_LIB", "default"), "steps": steps, "passes": passes,
    "share_of_all": {k: round(float(v / cyc.sum()), 4) for k, v in zip(PHASES, cyc)},
    "share_of_pass": {k: round(float(v / pass_total), 4) for k, v in per_pass.items()},
    "eval_share_of_pass": round(float((cyc[1] + cyc[3]) / pass_total), 4),
    "warp_cycles_per_pass": {**{k: round(float(v / passes / warps)) for k, v in per_pass.items()},
                             "pass": round(float(pass_total / passes / warps))},
    "serial_warp_cycles_per_pass": {k: round(float(v / passes / warps)) for k, v in zip(SERIAL, cyc[SER])},
    "serial_cycles_per_pass_on_its_warps": {k: round(float(v / passes)) for k, v in zip(SERIAL, cyc[SER])},
}))
