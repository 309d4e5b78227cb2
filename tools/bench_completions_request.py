#!/usr/bin/env python3
"""Measurement of the /v1/completions request path (schema completions-openai): the realistic code-completion / vLLM corpus of
tests/test_completions_request_cpu.py, replicated to --n bodies, through aigw_chat_translate_device (device-resident bodies, one
call per size class) and aigw_chat_translate_host (end to end from host buffers).  Prints one JSON line with bodies/s and GB/s of
input, the status / reason counts (token-id prompts beyond the index stage's capacity decline), the card's name and power limit,
and a CPU leg: the Python oracle (ParseBody verdict + the C++ sjson set) on a sample, single-threaded."""
import argparse, collections, json, os, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _completions_request_oracle as Q
import test_completions_request_cpu as G
import test_translate_edges_cpu as E
import aigw_b200 as A

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=100_000)
ap.add_argument("--distinct", type=int, default=2000)
ap.add_argument("--override", default="")
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--cpu-sample", type=int, default=500)
a = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power = [x.strip() for x in q.splitlines()[0].split(",")]
    return name, power


name, power = card()
ctx = A.Context(0)
cfg = ctx.cfg("completions-openai", model_override=a.override or None)
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
# ---- host call, end to end
arena, offs, lens = A.capi.pack_bodies(bodies)
for _ in range(a.warmup): ctx.chat_translate_host(cfg, arena, offs, lens)
t = time.perf_counter()
for _ in range(a.steps): res, _, _ = ctx.chat_translate_host(cfg, arena, offs, lens)
host_s = (time.perf_counter() - t) / a.steps
host_statuses = collections.Counter(zip(res["status"].tolist(), res["reason"].tolist()))
assert set(host_statuses) <= {(0, 0), (4, 5)}, host_statuses   # OK, or declined for token capacity
# ---- CPU oracle, single thread
sample = distinct[:a.cpu_sample]
t = time.perf_counter()
for b in sample: Q.translate(b, a.override)
cpu_s = time.perf_counter() - t
print(json.dumps({"workload": "completions-request", "bodies": a.n, "distinct": a.distinct, "override": a.override, "mean_body_bytes": round(total / a.n),
                  "device_bodies_per_s": round(a.n / dev_s), "device_GB_per_s": round(total / dev_s / 1e9, 3),
                  "host_e2e_bodies_per_s": round(a.n / host_s), "host_e2e_GB_per_s": round(total / host_s / 1e9, 3),
                  "oracle_1thread_bodies_per_s": round(len(sample) / cpu_s), "device_status": {"%d/%d" % k: v for k, v in sorted(statuses.items())},
                  "host_status": {"%d/%d" % k: v for k, v in sorted(host_statuses.items())}, "gpu": name, "power_limit": power}))
ctx.close()
