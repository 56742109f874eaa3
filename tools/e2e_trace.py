"""Timeline of the end-to-end call (PLSVO_TRACE_E2E=1, stderr of the library) on bench.py's lean inputs, plus the
single-shot breakdown (upload / kernel / download, each synchronised)."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import torch
import plsvo_b200
from plsvo_b200 import synth
import bench
B = int(os.environ.get("TUNE_B", 1024))
dev = torch.device("cuda", 0)
data = synth.make_align_batch(batch=B, n_pts=300, n_segs=80, device=dev, seed=3000)
data, nbytes, keep = bench.lean_copy(data, torch)
stream = torch.cuda.Stream(dev); torch.cuda.set_stream(stream)
ctx = plsvo_b200.Context(0, stream.cuda_stream)
al = plsvo_b200.SparseImgAlign(4, 2, 30, ctx=ctx)
for _ in range(3): al.run(data)
for gate in os.environ.get("TRACE_GATES", "256").split(","):
    os.environ["PLSVO_GATE_CHUNK"] = gate
    for _ in range(2): al.run(data)
    os.environ["PLSVO_TRACE_E2E"] = "1"
    t0 = time.perf_counter()
    for _ in range(3): al.run(data)
    dt = (time.perf_counter() - t0) / 3
    os.environ.pop("PLSVO_TRACE_E2E")
    t0 = time.perf_counter()
    for _ in range(10): al.run(data)
    dt10 = (time.perf_counter() - t0) / 10
    print(json.dumps({"gate": gate, "ms_traced": round(dt * 1e3, 3), "ms": round(dt10 * 1e3, 3), "pairs_per_s": round(B / dt10), "bytes": nbytes}), flush=True)
for _ in range(2):
    t0 = time.perf_counter(); al.upload(data); ctx.sync(); t1 = time.perf_counter(); al.launch(); ctx.sync(); t2 = time.perf_counter(); al.download(); t3 = time.perf_counter()
print(json.dumps({"single_shot": {"upload_ms": round((t1-t0)*1e3,3), "h2d_gbs": round(nbytes/(t1-t0)/1e9, 1), "kernel_ms": round((t2-t1)*1e3,3), "download_ms": round((t3-t2)*1e3,3)}}))
