#!/usr/bin/env python3
"""Secondary bench — S2: Bedrock ConverseStream eventstream → OpenAI SSE back-translation.
Prints one JSON line in bench.py's shape (resident `value`, host-buffer `e2e`, roofline of the two kernels, CPU oracle baseline)."""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _workload as W
import _oracle as O
import aigw_b200 as A

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=200_000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--cpu-streams", type=int, default=50_000)
a = ap.parse_args()
ctx = A.Context(0)
base_n = 2000
arr, off, streams = W.bedrock_stream_corpus(base_n, seed=21)
reps = (a.streams + base_n - 1) // base_n
n = reps * base_n
buf = np.tile(arr, reps)
soff = np.concatenate([[0], np.tile(np.diff(off.astype(np.int64)), reps).cumsum()]).astype(np.uint64)
nbytes = int(soff[-1])
frames = sum(s.count(b":event-type") for s in streams) * reps
from bench import host_cores
ncpu = host_cores()   # affinity mask ∩ cgroup CPU quota
ns = min(a.cpu_streams, n)
tot = C.c_uint64(0)
L = O.lib(); L.oracle_bedrock_stream_batch.restype = C.c_double
L.oracle_bedrock_stream_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_char_p, C.c_int64, C.c_int, C.POINTER(C.c_uint64)]
sec = L.oracle_bedrock_stream_batch(buf.ctypes.data, soff.ctypes.data, ns, b"m", b"r", 7, ncpu, C.byref(tot))
cpu_rate = ns / sec
sec1 = L.oracle_bedrock_stream_batch(buf.ctypes.data, soff.ctypes.data, min(ns, 4000), b"m", b"r", 7, 1, C.byref(tot))
cpu1 = min(ns, 4000) / sec1
out_cap = 3 * nbytes
d_b = ctx.dalloc(nbytes + 64); d_o = ctx.dalloc(soff.nbytes); d_out = ctx.dalloc(out_cap); d_r = ctx.dalloc(n * 64); d_u = ctx.dalloc(64)
ctx.h2d(d_b, buf); ctx.h2d(d_o, soff)
run = lambda: ctx.bedrock_stream_device(d_b, d_o, n, nbytes, d_out, out_cap, d_r, d_u, request_model="m", response_id="r", created=7)
for _ in range(a.warmup): run()
ctx.sync(); ms = [run() for _ in range(a.steps)]; ctx.sync()
res = np.zeros(n, dtype=A.capi.StreamResult); ctx.d2h(res, d_r)
assert (res["status"] == 0).all()
out_bytes = int(res["out_len"].sum())
step_s = float(np.mean(ms)) / 1e3
alg = nbytes + out_bytes + n * 64
pin, pp = ctx.host_array(nbytes + 64); pin[:nbytes] = buf
for _ in range(2): ctx.bedrock_stream_host(pin[:nbytes], soff, "m", "r", 7)
t = time.perf_counter()
for _ in range(a.steps): r2, o2, st = ctx.bedrock_stream_host(pin[:nbytes], soff, "m", "r", 7)
e_wall = time.perf_counter() - t
assert (r2["status"] == 0).all() and int(r2["out_len"].sum()) == out_bytes
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
print(json.dumps({"metric": "Bedrock streams/sec, eventstream -> OpenAI SSE", "value": n / step_s, "unit": "streams/s", "n_gpus": 1, "steps": a.steps, "warmup": a.warmup,
                  "ms_per_step": step_s * 1e3, "higher_is_better": True, "dtype": "u8", "data": "synthetic",
                  "config": {"workload": f"{n} ConverseStream responses, mean {nbytes // n} B / {frames // n} frames (plain/tools/reasoning/cache mix, seed 21 tiled)", "bytes_in": nbytes, "bytes_out": out_bytes,
                             "frames_per_s": frames / step_s},
                  "roofline": {"bound": "hbm", "achieved": alg / step_s / 1e9, "peak": peak, "unit": "GB/s", "frac": alg / step_s / 1e9 / peak, "traffic": None, "kernel": "bedrock_frames_kernel + bedrock_emit_kernel"},
                  "e2e": {"value": n * a.steps / e_wall, "unit": "streams/s", "h2d_bytes_per_step": st["h2d_bytes"], "d2h_bytes_per_step": st["d2h_bytes"]},
                  "cpu_baseline": {"value": cpu_rate, "unit": "streams/s", "cores": ncpu, "kind": "port", "sample": f"{ns} streams, {ncpu} threads; single thread {cpu1:.0f} streams/s"}}))
