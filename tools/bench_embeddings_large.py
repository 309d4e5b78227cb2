"""Throughput and latency of aigw_embeddings_translate_large_* on the large realistic embeddings corpus
(tests/test_embeddings_large_cpu.py), per target: OpenAI with a model override, GCP Vertex AI, Amazon Titan.  Prints one JSON
line per measurement, each with the card's name and power limit read in the same run.  Needs an H100; there is no CPU path."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def emit(**kw):
    kw["card"] = CARD
    print(json.dumps(kw), flush=True)


def ctas(ctx, max_len):
    """the call's grid: 2 CTAs per SM, fewer when one workspace slice per CTA (sized by the longest request) would pass 1 GiB
    (emb_large_slice_bytes / emb_large_grid)"""
    tc, ec = max_len // 2 + 1024, max_len // 4 + 1024
    slice_ = ((tc * 4 + 15) // 16 * 16 + ec * 16 + 2 * tc * 16 + (tc + 15) // 16 * 16 + 65536 + 64 + 255) // 256 * 256
    return max(1, min((1 << 30) // slice_, 2 * ctx.sm_count))


def device_call(ctx, c, bodies, reps=10):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    cap = sum(4 * len(b) + 4096 for b in bodies)
    d_b, d_o, d_l, d_out, d_r, d_u = (ctx.dalloc(max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, cap, n * 32, 8))
    try:
        ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens)
        ms = []
        for i in range(reps + 2):
            ctx.memset(d_u, 0, 8)
            t = ctx.embeddings_translate_large_device(c, d_b, d_o, d_l, n, int(lens.max()), d_out, cap, d_r, d_u)
            if i >= 2:
                ms.append(t)
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, d_u)
        return float(np.median(ms)), int(used[0])
    finally:
        for d in (d_b, d_o, d_l, d_out, d_r, d_u):
            ctx.dfree(d)


def profile_split(ctx, targets):
    """the kernel time of each target's device call from torch.profiler's CUDA activity trace (a pass of its own)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    for name, (schema, override, bodies) in targets.items():
        c = ctx.cfg(schema, model_override=override)
        device_call(ctx, c, bodies, reps=1)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            device_call(ctx, c, bodies, reps=3)
        for e in prof.key_averages():
            if "emb_large_kernel" in e.key or "memset" in e.key.lower():
                t = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0)
                emit(what="profile", target=name, kernel=e.key[:60], calls=e.count, mean_ms=round(t / max(1, e.count) / 1e3, 3))


def main():
    import aigw_b200 as A
    import _oracle as O
    import test_embeddings_large_cpu as L
    ctx = A.Context(0)
    corpus = L.large_corpus()
    targets = {
        "openai+override": ("emb-openai", "text-embedding-005", corpus),
        "vertex": ("emb-gcp-vertexai", None, [b for b in corpus if not (isinstance(json.loads(b)["input"], list) and isinstance(json.loads(b)["input"][0], (int, list)))]),
        "titan": ("emb-aws-bedrock", None, [b for b in corpus if isinstance(json.loads(b)["input"], str)] + L.titan_bodies()),
    }
    if "--profile" in sys.argv:
        profile_split(ctx, targets)
        ctx.close()
        return
    for name, (schema, override, bodies) in targets.items():
        c = ctx.cfg(schema, model_override=override)
        ms, used = device_call(ctx, c, bodies)
        nbytes = sum(map(len, bodies))
        emit(what="device_call", target=name, requests=len(bodies), request_bytes=nbytes, output_bytes=used, ms=round(ms, 3),
             requests_per_s=round(len(bodies) / ms * 1e3), gb_per_s=round((nbytes + used) / ms / 1e6, 1), max_len=max(map(len, bodies)),
             ctas=ctas(ctx, max(map(len, bodies))))
        arena, offs, lens = A.pack_bodies(bodies)
        ctx.embeddings_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.embeddings_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="host_call", target=name, ms=round(1e3 * float(np.median(t)), 2), requests_per_s=round(len(bodies) / float(np.median(t))))
    # single requests: wall latency of one host call
    c = ctx.cfg("emb-gcp-vertexai")
    for size in (128 << 10, 1 << 20, 4 << 20):
        items = ",".join('"chunk %d %s \\u00e9"' % (i, "x" * 500) for i in range(size // 520))
        b = ('{"model":"text-embedding-004","input":[%s]}' % items).encode()
        arena, offs, lens = A.pack_bodies([b])
        t = []
        for i in range(60):
            t0 = time.perf_counter(); ctx.embeddings_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        t = np.array(t[10:]) * 1e6
        emit(what="single_request_wall_us", bytes=len(b), p50=round(float(np.percentile(t, 50))), p99=round(float(np.percentile(t, 99))))
    # BASELINE config 3's request shape (1 024 inputs of 64 characters) translated to Vertex
    rng = np.random.default_rng(3)
    shape3 = [json.dumps({"model": "text-embedding-3-small", "input": ["".join(chr(97 + int(x)) for x in rng.integers(0, 26, 64)) for _ in range(1024)]}).encode() for _ in range(2000)]
    ms, used = device_call(ctx, c, shape3)
    emit(what="config3_shape_vertex_device_call", requests=len(shape3), mean_bytes=int(np.mean([len(b) for b in shape3])), ms=round(ms, 3),
         requests_per_s=round(len(shape3) / ms * 1e3))
    # the oracle on one thread
    t0 = time.perf_counter(); nb = 0
    for b in corpus[:20]:
        O.embeddings_translate("gcp-vertexai", b); nb += len(b)
    emit(what="oracle_one_thread", mb_per_s=round(nb / (time.perf_counter() - t0) / 1e6, 1))
    # the serial walk's worst case: a 16 MiB - 1 body whose tokens sit in item objects, or in an unknown member
    n = (16 << 20) - 1
    # (0.4 tokens per byte: within the len / 2 + 1024 token cap)
    items = b'{"model":"m","input":[' + b",".join([b'{"content":"aaaaaaaaaaaa","x":[1111,2222]}'] * ((n - 64) // 43)) + b"]}"
    unknown = b'{"model":"m","input":"a","meta":[' + b",".join([b"1111"] * ((n - 64) // 5)) + b"]}"
    for label, b in (("items", items), ("unknown_member", unknown)):
        b = b + b" " * (n - len(b))
        ms, _ = device_call(ctx, c, [b], reps=3)
        g = ctx.embeddings_translate_large(c, [b])[0]
        emit(what="serial_walk_worst_case", layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))
    ctx.close()


CARD = "unknown"
if __name__ == "__main__":
    CARD = card()
    main()
