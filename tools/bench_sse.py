#!/usr/bin/env python3
"""Secondary bench — BASELINE.json configs[3]: SSE streamed response parse, 100k streams x 256 chunks x 80 B,
OpenAI-schema usage extract (S1 + C1).  Prints one JSON line in bench.py's shape (resident `value`, host-buffer `e2e`,
roofline of sse_usage_kernel, CPU oracle baseline)."""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _workload as W
import _oracle as O
import aigw_b200 as A

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=100_000)
ap.add_argument("--chunks", type=int, default=256)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--cpu-streams", type=int, default=20_000)
a = ap.parse_args()
ctx = A.Context(0)
buf, coff, cfirst = W.sse_corpus(4, 0, a.streams, chunks=a.chunks)
nbytes = int(coff[-1]); nchunks = len(coff) - 1
from bench import host_cores
ncpu = host_cores()   # affinity mask ∩ cgroup CPU quota
# CPU oracle (chunk-by-chunk replay) on a bounded sample
ns = min(a.cpu_streams, a.streams)
outu = np.zeros(ns, dtype=np.dtype([(k, "<u4") for k in ("input", "output", "total", "cached", "cache_creation", "reasoning", "mask")]))
sec = O.lib().oracle_sse_batch(buf.ctypes.data, coff.ctypes.data, cfirst.ctypes.data, ns, ncpu, outu.ctypes.data)
cpu_rate = ns * a.chunks / sec
# device-resident
d_b = ctx.dalloc(nbytes + 64); d_c = ctx.dalloc(coff.nbytes); d_f = ctx.dalloc(cfirst.nbytes); d_r = ctx.dalloc(a.streams * 48)
ctx.h2d(d_b, buf[: nbytes + 64] if len(buf) >= nbytes + 64 else buf); ctx.h2d(d_c, coff); ctx.h2d(d_f, cfirst)
for _ in range(a.warmup): ctx.sse_usage_device(d_b, d_c, d_f, a.streams, d_r)
ctx.sync(); ms = [ctx.sse_usage_device(d_b, d_c, d_f, a.streams, d_r) for _ in range(a.steps)]; ctx.sync()
res = np.zeros(a.streams, dtype=A.SseResult); ctx.d2h(res, d_r)
assert (res["status"] == 0).all()
# parity on the CPU sample
m = res["mask"][:ns]
assert (res["input"][:ns] == outu["input"]).all() and (res["total"][:ns] == outu["total"]).all() and (m == outu["mask"]).all()
step_s = float(np.mean(ms)) / 1e3
alg = nbytes + a.streams * 48
# host-buffer e2e
pin, pp = ctx.host_array(nbytes + 64); pin[:nbytes] = buf[:nbytes]
for _ in range(2): ctx.sse_usage_host(pin, coff, cfirst)
t = time.perf_counter()
for _ in range(a.steps): r2, st = ctx.sse_usage_host(pin, coff, cfirst)
e_wall = time.perf_counter() - t
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
print(json.dumps({"metric": "SSE chunks/sec, OpenAI usage extract", "value": nchunks / step_s, "unit": "chunks/s", "n_gpus": 1, "steps": a.steps, "warmup": a.warmup,
                  "ms_per_step": step_s * 1e3, "higher_is_better": True, "dtype": "u8", "data": "synthetic",
                  "config": {"workload": f"configs[3]: {a.streams} streams x {a.chunks} chunks x ~80 B, 20% ragged chunking, seed 4", "bytes": nbytes},
                  "roofline": {"bound": "hbm", "achieved": alg / step_s / 1e9, "peak": peak, "unit": "GB/s", "frac": alg / step_s / 1e9 / peak, "traffic": None, "kernel": "sse_usage_kernel"},
                  "e2e": {"value": nchunks * a.steps / e_wall, "unit": "chunks/s", "h2d_bytes_per_step": st["h2d_bytes"], "d2h_bytes_per_step": st["d2h_bytes"]},
                  "cpu_baseline": {"value": cpu_rate, "unit": "chunks/s", "cores": ncpu, "kind": "port", "sample": f"{ns} streams, {ncpu} threads"}}))
