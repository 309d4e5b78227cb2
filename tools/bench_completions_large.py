"""Throughput and latency of aigw_completions_translate_large_* on the large requests of tests/test_completions_large_cpu.py: the
device call (CUDA events, median of 10) with and without the model override, the kernel's own time from torch.profiler in a pass of
its own, the host call end to end, single-request wall latency of a fill-in-the-middle string prompt and a token-id prompt of the
same size (about 190 KB, 770 KB and 4 MB), and the serial worst cases at 16 MiB - 1.  Prints one JSON line per measurement, each
with the card's name, power limit and top SM clock read in the same run.  Needs an H100; there is no CPU path."""
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
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q.splitlines()[0] if q else "unknown"


def emit(**kw):
    kw["card"] = CARD
    print(json.dumps(kw), flush=True)


class Staged:
    """the bodies, tables and output arena of one device call, in device memory"""

    def __init__(self, ctx, bodies):
        import aigw_b200 as A
        self.ctx = ctx
        arena, offs, lens = A.pack_bodies(bodies)
        self.n, self.max_len = len(bodies), int(lens.max())
        self.cap = sum(len(b) + 512 for b in bodies)
        self.ptrs = [ctx.dalloc(max(16, x)) for x in (arena.nbytes + 64, offs.nbytes, lens.nbytes, self.cap, self.n * 32, 8)]
        ctx.h2d(self.ptrs[0], arena); ctx.h2d(self.ptrs[1], offs); ctx.h2d(self.ptrs[2], lens)

    def call(self, c, timed=True):
        d_b, d_o, d_l, d_out, d_r, d_u = self.ptrs
        self.ctx.memset(d_u, 0, 8)
        return self.ctx.completions_translate_large_device(c, d_b, d_o, d_l, self.n, self.max_len, d_out, self.cap, d_r, d_u, timed=timed)

    def used(self):
        u = np.zeros(1, dtype=np.uint64); self.ctx.d2h(u, self.ptrs[5]); return int(u[0])

    def free(self):
        for d in self.ptrs:
            self.ctx.dfree(d)


def device_ms(st, c, reps=10):
    ms = [st.call(c) for _ in range(reps + 2)][2:]
    return float(np.median(ms))


def profiler_kernel_ms(st, c, reps=10):
    """the kernel's own duration from torch.profiler's CUDA activity, median over reps untimed calls"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    st.call(c, timed=False); st.ctx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            st.call(c, timed=False)
        st.ctx.sync()
        torch.cuda.synchronize()
    ds = [e.device_time for e in prof.events() if "completions_large_kernel" in e.name]
    return float(np.median(ds)) / 1e3 if ds else float("nan"), len(ds)


def fim_body(size):
    """a compact fill-in-the-middle request of about `size` bytes: source text in prompt and suffix"""
    import random
    import test_completions_large_cpu as L
    r = random.Random(size)
    return json.dumps({"model": "qwen2.5-coder-7b", "prompt": L._source(r, size * 3 // 4), "suffix": L._source(r, size // 4),
                       "max_tokens": 64, "temperature": 0.2, "stream": True}, separators=(",", ":")).encode()


def token_body(size):
    """a compact token-id request of about `size` bytes: ids of 0-200 000, about 7 bytes each"""
    import random
    r = random.Random(size)
    return json.dumps({"model": "qwen2.5-coder-7b", "prompt": [r.randint(0, 200_000) for _ in range(size // 7)],
                       "max_tokens": 64, "temperature": 0.2, "stream": True}, separators=(",", ":")).encode()


def wall_us(ctx, c, b, reps=60):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies([b])
    t = []
    for _ in range(reps):
        t0 = time.perf_counter(); ctx.completions_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
    return np.array(t[10:]) * 1e6


def main():
    import aigw_b200 as A
    import test_completions_large_cpu as L
    ctx = A.Context(0)
    corpus = list(L.realistic_corpus())
    nbytes = sum(map(len, corpus))
    st = Staged(ctx, corpus)
    for name, override in (("no_override", None), ("override", "gpt-4-turbo")):
        c = ctx.cfg("completions-openai", model_override=override)
        got = ctx.completions_translate_large(c, corpus)
        assert all(g["status"] == A.AIGW_OK for g in got), [(g["status"], g["reason"]) for g in got]
        ms = device_ms(st, c)
        emit(what="device_call", target=name, requests=len(corpus), request_bytes=nbytes, output_bytes=st.used(), ms=round(ms, 3),
             gb_per_s_in=round(nbytes / ms / 1e6, 2), max_len=max(map(len, corpus)))
        kms, nk = profiler_kernel_ms(st, c)
        emit(what="kernel_profiler", target=name, launches=nk, ms=round(kms, 3))
        arena, offs, lens = A.pack_bodies(corpus)
        ctx.completions_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.completions_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="host_call", target=name, ms=round(1e3 * float(np.median(t)), 2), gb_per_s_in=round(nbytes / float(np.median(t)) / 1e9, 2))
    st.free()
    # single requests: wall latency of one host call, a string prompt against a token-id prompt of about the same size, alternated
    c = ctx.cfg("completions-openai", model_override="gpt-4-turbo")
    for size in (190_000, 770_000, 4_000_000):
        pair = (("fim", fim_body(size)), ("token_ids", token_body(size)))
        for _, b in pair:
            assert ctx.completions_translate_large(c, [b])[0]["status"] == A.AIGW_OK
        walls = {k: [] for k, _ in pair}
        for _ in range(3):
            for k, b in pair:
                walls[k].append(wall_us(ctx, c, b, reps=30))
        for k, b in pair:
            t = np.concatenate(walls[k])
            one = Staged(ctx, [b])
            ms = device_ms(one, c)
            one.free()
            emit(what="single_request_wall_us", prompt=k, bytes=len(b), p50=round(float(np.percentile(t, 50))), p99=round(float(np.percentile(t, 99))),
                 kernel_ms=round(ms, 3))
    # the serial worst cases at 16 MiB - 1, each within the len / 2 + 1024 token cap: a flat id prompt (whole-CTA stage: no serial
    # pass), a batch of one-id arrays (the outer array is walked serially, each inner one is stepped over), and scalars inside
    # objects in an unknown member (the grammar pass visits every token)
    n = (16 << 20) - 1
    layouts = (("flat_id_prompt", '{"model":"m","prompt":[' + ",".join(["1111"] * ((n - 64) // 5)) + "]}"),
               ("one_id_batch", '{"model":"m","prompt":[' + ",".join(["[100000]"] * ((n - 64) // 9)) + "]}"),
               ("scalars_in_objects", '{"model":"m","prompt":"p","x":[' + ",".join(['{"a":100000000}'] * ((n - 64) // 16)) + "]}"))
    for label, s in layouts:
        b = s.encode()
        b = b + b" " * (n - len(b))
        one = Staged(ctx, [b])
        ms = device_ms(one, c, reps=3)
        one.free()
        g = ctx.completions_translate_large(c, [b])[0]
        emit(what="serial_worst_case", layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))
    ctx.close()


CARD = "unknown"
if __name__ == "__main__":
    CARD = card()
    main()
