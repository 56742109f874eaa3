"""A/B of the end-to-end alignment call on ONE frame-chain batch: two stacks (ref, cur; 2B frames over the link) against
one stack (PLSVO_ALIGN_FRAME_CHAIN; B + 1 frames), interleaved in blocks so that the drift of the host link's rate hits
both, with the library's own timeline (PLSVO_TRACE_E2E=1) of one call each.  Usage: python tools/e2e_chain_ab.py"""
import copy, json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import numpy as np
import torch
import plsvo_b200
from plsvo_b200 import numa, synth
import bench

B = int(os.environ.get("TUNE_B", 1024))
dev = torch.device("cuda", 0)
numa.bind_to_device(0)
full = synth.make_chain_batch(batch=B, n_pts=300, n_segs=80, device=dev, seed=7000)
two, bytes_two, keep = bench.lean_copy(full, torch)
ft = torch.from_numpy(synth.chain_frames(full, levels=[full.min_level])[full.min_level]).pin_memory()
one = copy.copy(two)
one.frame_pyr = {full.min_level: ft.numpy()}
bytes_one = bytes_two - sum(v.nbytes for v in two.ref_pyr.values()) - sum(v.nbytes for v in two.cur_pyr.values()) + ft.numpy().nbytes
stream = torch.cuda.Stream(dev); torch.cuda.set_stream(stream)
ctx = plsvo_b200.Context(0, stream.cuda_stream)
al = plsvo_b200.SparseImgAlign(4, 2, 30, ctx=ctx)
for _ in range(3):
    a = al.run(two); b = al.run(one)
assert np.array_equal(a.T_cur_w, b.T_cur_w) and np.array_equal(a.iters, b.iters)
times = {"two_stacks": [], "one_stack": []}
for rnd in range(int(os.environ.get("AB_ROUNDS", 4))):
    for name, d in (("two_stacks", two), ("one_stack", one)):
        for _ in range(8):
            t0 = time.perf_counter(); al.run(d); times[name].append(1e3 * (time.perf_counter() - t0))
os.environ["PLSVO_TRACE_E2E"] = "1"
for name, d in (("two_stacks", two), ("one_stack", one)):
    print("# trace", name, file=sys.stderr, flush=True)
    al.run(d)
os.environ.pop("PLSVO_TRACE_E2E")
res = {"pairs": B, "bytes": {"two_stacks": int(bytes_two), "one_stack": int(bytes_one)}}
for name, t in times.items():
    t = np.array(t)
    res[name] = {"ms_p50": round(float(np.median(t)), 3), "ms_min": round(float(t.min()), 3), "ms_p90": round(float(np.percentile(t, 90)), 3),
                 "pairs_per_s_p50": round(B / (np.median(t) * 1e-3))}
# launch-side knobs of the streamed call, re-examined for the one-stack form (fewer bytes: the link may no longer be the bound)
res["one_stack_knobs"] = {}
for label, env in (("variant_128_4", {"PLSVO_VARIANT": "128,4"}), ("variant_160_3", {"PLSVO_VARIANT": "160,3"}),
                   ("gate_chunk_128", {"PLSVO_GATE_CHUNK": "128"}), ("gate_chunk_512", {"PLSVO_GATE_CHUNK": "512"}),
                   ("default_again", {})):
    os.environ.update(env)
    for _ in range(2):
        al.run(one)
    t = []
    for _ in range(12):
        t0 = time.perf_counter(); al.run(one); t.append(1e3 * (time.perf_counter() - t0))
    for k in env:
        os.environ.pop(k)
    res["one_stack_knobs"][label] = {"ms_p50": round(float(np.median(t)), 3), "ms_min": round(float(min(t)), 3)}
# the plain sequence of the one-stack call: upload, kernel, download, each synchronised
for name, d in (("two_stacks", two), ("one_stack", one)):
    for _ in range(2):
        t0 = time.perf_counter(); al.upload(d); ctx.sync(); t1 = time.perf_counter(); al.launch(); ctx.sync(); t2 = time.perf_counter(); al.download(); t3 = time.perf_counter()
    res[name]["single_shot"] = {"upload_ms": round((t1 - t0) * 1e3, 3), "h2d_gbs": round(res["bytes"][name] / (t1 - t0) / 1e9, 1),
                                "kernel_ms": round((t2 - t1) * 1e3, 3), "download_ms": round((t3 - t2) * 1e3, 3)}
print(json.dumps(res))
