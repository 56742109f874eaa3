"""e2e (host buffers -> C ABI -> host results) timing vs the arrival gate's chunk size (PLSVO_GATE_CHUNK)."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import numpy as np, torch
import plsvo_b200
from plsvo_b200 import synth
B = int(os.environ.get("TUNE_B", 1024))
dev = torch.device("cuda", 0)
data = synth.make_align_batch(batch=B, n_pts=300, n_segs=80, device=dev, seed=3000)
keep = []
def pin(a):
    t = torch.from_numpy(a).pin_memory(); keep.append(t); return t.numpy()
for name in ("T_ref_w", "T_cur_w", "pt_px", "pt_f", "pt_pos", "seg_spx", "seg_epx", "seg_sf", "seg_ef", "seg_spos", "seg_epos", "seg_length"):
    setattr(data, name, pin(getattr(data, name)))
for pyr in (data.ref_pyr, data.cur_pyr):
    for l in list(pyr): pyr[l] = pin(pyr[l])
if os.environ.get("TUNE_LEAN", "1") == "1":  # what bench.py's e2e leg ships: finest level only + feature depths
    sys.path.insert(0, ROOT)
    import bench
    data, nbytes, keep2 = bench.lean_copy(data, torch)
    print(json.dumps({"lean_bytes_per_step": nbytes}))
ctx = plsvo_b200.Context(0)
al = plsvo_b200.SparseImgAlign(4, 2, 30, ctx=ctx)
for gate in (128, 256, 384, 512):
    os.environ['PLSVO_GATE_CHUNK'] = str(gate)
    for _ in range(3): al.run(data)
    t0 = time.perf_counter()
    n = 10
    for _ in range(n): al.run(data)
    dt = (time.perf_counter() - t0) / n
    print(json.dumps({"gate": gate, "ms": round(dt * 1e3, 3), "pairs_per_s": round(B / dt)}), flush=True)
# breakdown of the plain upload -> launch -> download sequence
t0 = time.perf_counter(); al.upload(data); ctx.sync(); t1 = time.perf_counter(); al.launch(); ctx.sync(); t2 = time.perf_counter(); al.download(); t3 = time.perf_counter()
print(json.dumps({"upload_ms": round((t1-t0)*1e3,3), "launch_ms": round((t2-t1)*1e3,3), "download_ms": round((t3-t2)*1e3,3)}))
