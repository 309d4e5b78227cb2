#!/usr/bin/env python3
"""Measurement of Cohere /v2/rerank (schema rerank-cohere): the realistic RAG rerank corpus of tests/test_rerank_cpu.py, replicated
to --n bodies, through aigw_chat_translate_device (device-resident bodies, one call per size class); the fused small-batch kernel's
wall latency (p50 of aigw_chat_translate_host over --reps calls of 1, 64 and 512 requests of at most 5120 bytes); the buffered
usage call aigw_rerank_response_usage_host on the response corpus; and a CPU leg: the Python oracle on a sample, single-threaded.
Prints one JSON line with the card's name and power limit."""
import argparse, collections, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _rerank_oracle as Q
import test_rerank_cpu as G
import test_translate_edges_cpu as E
import aigw_b200 as A

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=100_000)
ap.add_argument("--distinct", type=int, default=2000)
ap.add_argument("--override", default="")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--reps", type=int, default=200)
ap.add_argument("--cpu-sample", type=int, default=500)
a = ap.parse_args()

def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power = [x.strip() for x in q.splitlines()[0].split(",")]
    return name, power


name, power = card()
ctx = A.Context(0)
cfg = ctx.cfg("rerank-cohere", model_override=a.override or None, api_version="v2")
distinct = G.realistic_corpus(a.distinct)
bodies = [distinct[i % len(distinct)] for i in range(a.n)]
total = sum(len(b) for b in bodies)
# ---- device call: bodies resident on the device, grouped by size class, one call per class
by_cls = collections.defaultdict(list)
for b in bodies:
    by_cls[E.class_of(len(b))].append(b)
legs = []
for c, bs in sorted(by_cls.items()):
    arena, offs, lens = A.capi.pack_bodies(bs)
    n = len(bs); out_cap = 2 * int(lens.astype(np.int64).sum()) + 1024 * n + 4096
    d = [ctx.dalloc(arena.nbytes), ctx.dalloc(offs.nbytes), ctx.dalloc(lens.nbytes), ctx.dalloc(out_cap), ctx.dalloc(32 * n), ctx.dalloc(8)]
    ctx.h2d(d[0], arena); ctx.h2d(d[1], offs); ctx.h2d(d[2], lens)
    legs.append((c, n, d, out_cap))


def device_pass():
    for c, n, d, out_cap in legs:
        ctx.memset(d[5], 0, 8)
        ctx.chat_translate_device(cfg, d[0], d[1], d[2], n, c, d[3], out_cap, d[4], d[5], timed=False)
    ctx.sync()


for _ in range(a.warmup): device_pass()
t = time.perf_counter()
for _ in range(a.steps): device_pass()
dev_s = (time.perf_counter() - t) / a.steps
statuses = collections.Counter()
for c, n, d, _ in legs:
    res = np.zeros(n, dtype=A.DocResult); ctx.d2h(res, d[4])
    statuses.update(zip(res["status"].tolist(), res["reason"].tolist()))
    for p in d: ctx.dfree(p)
# ---- fused small-batch kernel: wall latency of one host call
small = [b for b in distinct if len(b) <= E.SMALL_MAX]
lat = {}
for k in (1, 64, 512):
    batch = [small[i % len(small)] for i in range(k)]
    arena, offs, lens = A.capi.pack_bodies(batch)
    for _ in range(10): ctx.chat_translate_host(cfg, arena, offs, lens)
    ts = []
    for _ in range(a.reps):
        t = time.perf_counter(); ctx.chat_translate_host(cfg, arena, offs, lens); ts.append(time.perf_counter() - t)
    lat[k] = round(float(np.median(ts)) * 1e6, 1)
# ---- buffered response usage, host call end to end
resp = G.response_corpus()
resp = [resp[i % len(resp)] for i in range(a.n)]
rtotal = sum(len(b) for b in resp)
arena, offs, lens = A.capi.pack_bodies(resp)
for _ in range(a.warmup): ctx.response_usage_host(arena, offs, lens, cost_types=(0, 3, 4), rerank=True)
t = time.perf_counter()
for _ in range(a.steps): ctx.response_usage_host(arena, offs, lens, cost_types=(0, 3, 4), rerank=True)
usage_s = (time.perf_counter() - t) / a.steps
# ---- CPU oracle, single thread
sample = distinct[:a.cpu_sample]
t = time.perf_counter()
for b in sample: Q.translate(b, a.override)
cpu_s = time.perf_counter() - t
t = time.perf_counter()
for b in resp[:a.cpu_sample * 4]: Q.response_usage(b)
cpu_usage_s = time.perf_counter() - t
print(json.dumps({"workload": "rerank", "bodies": a.n, "distinct": a.distinct, "override": a.override, "mean_body_bytes": round(total / a.n),
                  "device_bodies_per_s": round(a.n / dev_s), "device_GB_per_s": round(total / dev_s / 1e9, 3),
                  "fused_wall_p50_us": {str(k): v for k, v in lat.items()},
                  "usage_host_bodies_per_s": round(a.n / usage_s), "usage_mean_body_bytes": round(rtotal / a.n),
                  "oracle_1thread_request_bodies_per_s": round(len(sample) / cpu_s), "oracle_1thread_usage_bodies_per_s": round(a.cpu_sample * 4 / cpu_usage_s),
                  "device_status": {"%d/%d" % k: v for k, v in sorted(statuses.items())}, "gpu": name, "power_limit": power}))
ctx.close()
