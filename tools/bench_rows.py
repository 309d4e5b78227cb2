#!/usr/bin/env python3
"""Secondary bench for the widened rows: R1 (Bedrock buffered response → OpenAI JSON) and B1 (body mutation).
One JSON line per row in bench.py's shape (resident `value`, host-buffer `e2e`, roofline, CPU oracle baseline)."""
import argparse, ctypes as C, json, os, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _workload as W
import _oracle as O
import aigw_b200 as A
from aigw_b200 import capi

ap = argparse.ArgumentParser()
ap.add_argument("--n", type=int, default=1_000_000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=3)
ap.add_argument("--cpu-n", type=int, default=200_000)
ap.add_argument("--rows", default="r1,b1")
a = ap.parse_args()
ctx = A.Context(0)
from bench import host_cores
ncpu = host_cores()   # affinity mask ∩ cgroup CPU quota
peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
L = O.lib()


def tile(bodies, n):
    arena, offs, lens = capi.pack_bodies(bodies)
    reps = (n + len(bodies) - 1) // len(bodies)
    stride = int(offs[-1])
    big = np.tile(arena[:stride], reps)
    boffs = (np.tile(offs[:-1].astype(np.int64), reps) + np.repeat(np.arange(reps, dtype=np.int64) * stride, len(bodies))).astype(np.uint64)
    blens = np.tile(lens, reps)
    return big, np.concatenate([boffs, [np.uint64(reps * stride)]]).astype(np.uint64), blens.astype(np.uint32), reps * len(bodies)


def line(metric, unit, n, step_s, e_rate, st, alg, cpu_rate, cpu1, ns, workload, kernel, extra):
    print(json.dumps({"metric": metric, "value": n / step_s, "unit": unit, "n_gpus": 1, "steps": a.steps, "warmup": a.warmup, "ms_per_step": step_s * 1e3, "higher_is_better": True,
                      "dtype": "u8", "data": "synthetic", "config": dict({"workload": workload}, **extra),
                      "roofline": {"bound": "hbm", "achieved": alg / step_s / 1e9, "peak": peak, "unit": "GB/s", "frac": alg / step_s / 1e9 / peak, "traffic": None, "kernel": kernel},
                      "e2e": {"value": e_rate, "unit": unit, "h2d_bytes_per_step": st["h2d_bytes"], "d2h_bytes_per_step": st["d2h_bytes"]},
                      "cpu_baseline": {"value": cpu_rate, "unit": unit, "cores": ncpu, "kind": "port", "sample": f"{ns} bodies, {ncpu} threads; single thread {cpu1:.0f}/s"}}), flush=True)


if "r1" in a.rows:
    rng = np.random.default_rng(17)
    base = [W.bedrock_response_body(rng, ["plain", "tools", "reasoning", "cache"][i % 4]) for i in range(4000)]
    big, offs, lens, n = tile(base, a.n)
    nbytes = int(offs[-1]); ns = min(a.cpu_n, n)
    L.oracle_bedrock_response_batch.restype = C.c_double
    L.oracle_bedrock_response_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.POINTER(C.c_uint64)]
    # the batch helper takes contiguous offsets[i]..offsets[i+1]; bodies are 16-byte padded with spaces, which the decoder ignores
    tot = C.c_uint64(0)
    sec = L.oracle_bedrock_response_batch(big.ctypes.data, offs.ctypes.data, ns, ncpu, C.byref(tot)); cpu_rate = ns / sec
    n1 = min(ns, 20000); sec1 = L.oracle_bedrock_response_batch(big.ctypes.data, offs.ctypes.data, n1, 1, C.byref(tot)); cpu1 = n1 / sec1
    cfg = capi.Context.cfg("resp-aws-bedrock", model_override="anthropic.claude-3-sonnet"); cfg.response_id = b"2bc5b090-a26c-4007-9467-ce5adc4ffa1d"; cfg.created = 1731679200
    out_cap = 2 * nbytes + 256 * n
    d_b = ctx.dalloc(nbytes + 64); d_o = ctx.dalloc(offs.nbytes); d_l = ctx.dalloc(lens.nbytes); d_out = ctx.dalloc(out_cap); d_r = ctx.dalloc(n * 32); d_u = ctx.dalloc(64)
    ctx.h2d(d_b, big); ctx.h2d(d_o, offs[:-1].copy()); ctx.h2d(d_l, lens)
    ml = int(lens.max())
    def run():
        ctx.memset(d_u, 0, 8)
        return ctx.chat_translate_device(cfg, d_b, d_o, d_l, n, ml, d_out, out_cap, d_r, d_u)
    for _ in range(a.warmup): run()
    ctx.sync(); ms = [run() for _ in range(a.steps)]; ctx.sync()
    res = np.zeros(n, dtype=A.DocResult); ctx.d2h(res, d_r)
    assert (res["status"] == 0).all(), np.bincount(res["reason"])
    out_bytes = int(res["body_len"].sum()) + 32 * n
    step_s = float(np.mean(ms)) / 1e3
    pin, pp = ctx.host_array(nbytes + 64); pin[:nbytes] = big[:nbytes]
    o2 = offs[:-1].copy()
    for _ in range(2): ctx.chat_translate_host(cfg, pin, o2, lens)
    t = time.perf_counter()
    for _ in range(a.steps): r2, oo, st = ctx.chat_translate_host(cfg, pin, o2, lens)
    e_wall = time.perf_counter() - t
    assert (r2["status"] == 0).all()
    line("Bedrock Converse responses/sec -> OpenAI ChatCompletionResponse", "bodies/s", n, step_s, n * a.steps / e_wall, st, nbytes + out_bytes, cpu_rate, cpu1, ns,
         f"{n} buffered Converse responses, mean {int(lens.mean())} B (text / tool-use / reasoning / cache-usage mix, seed 17 tiled)", "chat_index + chat_walk + chat_emit (response direction)",
         {"bytes_in": nbytes, "bytes_out": out_bytes})
    for p in (d_b, d_o, d_l, d_out, d_r, d_u): ctx.dfree(p)

if "b1" in a.rows:
    arena0, offs0, lens0 = W.chat_corpus(2, 0, 20000)
    base = [bytes(arena0[int(offs0[i]):int(offs0[i]) + int(lens0[i])]) for i in range(20000)]
    big, offs, lens, n = tile(base, a.n)
    nbytes = int(offs[-1]); ns = min(a.cpu_n, n)
    rm = ["stream_options"]; st_ = [("temperature", "0.5"), ("max_tokens", "150"), ("custom_field", "\"route-level-value\"")]
    L.oracle_body_mutate_batch.restype = C.c_double
    L.oracle_body_mutate_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.POINTER(C.c_uint64)]
    crm = (C.c_char_p * 1)(*[r.encode() for r in rm]); csp = (C.c_char_p * 3)(*[p.encode() for p, _ in st_]); csv = (C.c_char_p * 3)(*[v.encode() for _, v in st_])
    # the oracle batch reads offsets[i]..offsets[i+1]: give it exact lengths through a packed copy of the sample
    samp = b"".join(base[i % len(base)] for i in range(ns)); soff = np.zeros(ns + 1, dtype=np.uint64); np.cumsum([len(base[i % len(base)]) for i in range(ns)], out=soff[1:])
    sbuf = np.frombuffer(samp, dtype=np.uint8)
    tot = C.c_uint64(0)
    sec = L.oracle_body_mutate_batch(sbuf.ctypes.data, soff.ctypes.data, ns, crm, 1, csp, csv, 3, ncpu, C.byref(tot)); cpu_rate = ns / sec
    n1 = min(ns, 20000); sec1 = L.oracle_body_mutate_batch(sbuf.ctypes.data, soff.ctypes.data, n1, crm, 1, csp, csv, 3, 1, C.byref(tot)); cpu1 = n1 / sec1
    out_cap = nbytes + 128 * n
    d_b = ctx.dalloc(nbytes + 64); d_o = ctx.dalloc(offs.nbytes); d_l = ctx.dalloc(lens.nbytes); d_out = ctx.dalloc(out_cap); d_r = ctx.dalloc(n * 16); d_u = ctx.dalloc(64)
    ctx.h2d(d_b, big); ctx.h2d(d_o, offs[:-1].copy()); ctx.h2d(d_l, lens)
    ml = int(lens.max())
    run = lambda: ctx.body_mutate_device(rm, st_, d_b, d_o, d_l, n, ml, d_out, out_cap, d_r, d_u)
    for _ in range(a.warmup): run()
    ctx.sync(); ms = [run() for _ in range(a.steps)]; ctx.sync()
    res = np.zeros(n, dtype=capi.MutResult); ctx.d2h(res, d_r)
    assert (res["status"] == 0).all(), np.bincount(res["reason"])
    out_bytes = int(res["out_len"].sum())
    step_s = float(np.mean(ms)) / 1e3
    pin, pp = ctx.host_array(nbytes + 64); pin[:nbytes] = big[:nbytes]
    o2 = offs[:-1].copy()
    for _ in range(2): ctx.body_mutate_host(rm, st_, pin, o2, lens)
    t = time.perf_counter()
    for _ in range(a.steps): r2, oo, st = ctx.body_mutate_host(rm, st_, pin, o2, lens)
    e_wall = time.perf_counter() - t
    assert (r2["status"] == 0).all()
    line("body mutations/sec (1 remove + 3 set, top-level)", "bodies/s", n, step_s, n * a.steps / e_wall, st, nbytes + out_bytes, cpu_rate, cpu1, ns,
         f"{n} ChatCompletion bodies of the C2 corpus (~4 KB), mutation of tests/data-plane/extproc_test.go:71-83", "body_mutate_kernel", {"bytes_in": nbytes, "bytes_out": out_bytes})

if "sha" in a.rows:
    # SigV4 payload hash of translated Bedrock bodies (aws.go:93-117): 1 M bodies of ~4.1 KB, device-resident spans
    arena0, offs0, lens0 = W.chat_corpus(2, 0, 20000)
    base = [O.chat_translate("aws-bedrock", bytes(arena0[int(offs0[i]):int(offs0[i]) + int(lens0[i])])).body for i in range(20000)]
    big, offs, lens, n = tile(base, a.n)
    nbytes = int(offs[-1]); ns = min(a.cpu_n, n)
    L.oracle_sha256_batch.restype = C.c_double
    L.oracle_sha256_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    dg = np.zeros((ns, 32), dtype=np.uint8)
    sec = L.oracle_sha256_batch(big.ctypes.data, offs.ctypes.data, lens.ctypes.data, ns, ncpu, dg.ctypes.data); cpu_rate = ns / sec
    n1 = min(ns, 20000); sec1 = L.oracle_sha256_batch(big.ctypes.data, offs.ctypes.data, lens.ctypes.data, n1, 1, dg.ctypes.data); cpu1 = n1 / sec1
    d_b = ctx.dalloc(nbytes + 64); d_o = ctx.dalloc(offs.nbytes); d_l = ctx.dalloc(lens.nbytes); d_d = ctx.dalloc(n * 32)
    ctx.h2d(d_b, big); ctx.h2d(d_o, offs[:-1].copy()); ctx.h2d(d_l, lens)
    run = lambda: ctx.sha256_device(d_b, d_o, d_l, n, d_d)
    for _ in range(a.warmup): run()
    ctx.sync(); ms = [run() for _ in range(a.steps)]; ctx.sync()
    dig = np.zeros((n, 32), dtype=np.uint8); ctx.d2h(dig, d_d)
    assert (dig[:ns] == dg).all()
    step_s = float(np.mean(ms)) / 1e3
    msg_bytes = int(lens.astype(np.int64).sum())
    print(json.dumps({"metric": "SigV4 payload SHA-256, bodies/sec", "value": n / step_s, "unit": "bodies/s", "n_gpus": 1, "steps": a.steps, "warmup": a.warmup, "ms_per_step": step_s * 1e3,
                      "higher_is_better": True, "dtype": "u32", "data": "synthetic", "config": {"workload": f"{n} translated Bedrock bodies, mean {msg_bytes // n} B", "bytes_in": msg_bytes},
                      "roofline": {"bound": "integer pipe (≈ 2.9 k instructions per 64-byte block); HBM shown for scale", "achieved": (msg_bytes + 32 * n) / step_s / 1e9, "peak": peak, "unit": "GB/s",
                                   "frac": (msg_bytes + 32 * n) / step_s / 1e9 / peak, "traffic": None, "kernel": "sha256_kernel"},
                      "cpu_baseline": {"value": cpu_rate, "unit": "bodies/s", "cores": ncpu, "kind": "port", "sample": f"{ns} bodies, {ncpu} threads; single thread {cpu1:.0f}/s (portable C, no SHA-NI)"}}), flush=True)
