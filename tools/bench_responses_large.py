"""Throughput and latency of aigw_responses_translate_large_* on the long agent sessions of tests/test_responses_large_cpu.py: the
device call (CUDA events, median of 10) with and without the model override, the kernel's own time from torch.profiler in a pass of
its own, the host call end to end, single-request wall latency at about 128 KiB, 1 MiB and 4 MiB, and the serial walk's worst case.
Prints one JSON line per measurement, each with the card's name, power limit and top SM clock read in the same run.  Needs an H100;
there is no CPU path."""
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
        return self.ctx.responses_translate_large_device(c, d_b, d_o, d_l, self.n, self.max_len, d_out, self.cap, d_r, d_u, timed=timed)

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
    ds = [e.device_time for e in prof.events() if "responses_large_kernel" in e.name]
    return float(np.median(ds)) / 1e3 if ds else float("nan"), len(ds)


def main():
    import aigw_b200 as A
    import test_responses_large_cpu as L
    ctx = A.Context(0)
    corpus = list(L.realistic_corpus())
    nbytes = sum(map(len, corpus))
    st = Staged(ctx, corpus)
    for name, override in (("no_override", None), ("override", "gpt-5-mini")):
        c = ctx.cfg("responses-openai", model_override=override)
        got = ctx.responses_translate_large(c, corpus)
        assert all(g["status"] == A.AIGW_OK for g in got), [(g["status"], g["reason"]) for g in got]
        ms = device_ms(st, c)
        emit(what="device_call", target=name, requests=len(corpus), request_bytes=nbytes, output_bytes=st.used(), ms=round(ms, 3),
             gb_per_s_in=round(nbytes / ms / 1e6, 2), max_len=max(map(len, corpus)))
        kms, nk = profiler_kernel_ms(st, c)
        emit(what="kernel_profiler", target=name, launches=nk, ms=round(kms, 3))
        arena, offs, lens = A.pack_bodies(corpus)
        ctx.responses_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.responses_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="host_call", target=name, ms=round(1e3 * float(np.median(t)), 2), gb_per_s_in=round(nbytes / float(np.median(t)) / 1e9, 2))
    st.free()
    # single requests: wall latency of one host call
    c = ctx.cfg("responses-openai", model_override="gpt-5-mini")
    for size in (128 << 10, 1 << 20, 4 << 20):
        b = L.long_session(77, size)
        arena, offs, lens = A.pack_bodies([b])
        assert ctx.responses_translate_large(c, [b])[0]["status"] == A.AIGW_OK
        t = []
        for i in range(60):
            t0 = time.perf_counter(); ctx.responses_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        t = np.array(t[10:]) * 1e6
        one = Staged(ctx, [b])
        ms = device_ms(one, c)
        one.free()
        emit(what="single_request_wall_us", bytes=len(b), p50=round(float(np.percentile(t, 50))), p99=round(float(np.percentile(t, 99))), kernel_ms=round(ms, 3))
    # the serial walk's worst case at 16 MiB - 1: scalars in an ignored member (the grammar pass alone), and tiny input items
    # (the member walk visits every one)
    n = (16 << 20) - 1
    flat = '{"model":"m","x":[' + ",".join(["1111"] * ((n - 64) // 5)) + "]}"
    item = '{"role":"user","content":"h"}'
    items = '{"model":"m","input":[' + ",".join([item] * ((n - 64) // (len(item) + 1))) + "]}"
    for label, s in (("ignored_member_scalars", flat), ("tiny_input_items", items)):
        b = s.encode()
        b = b + b" " * (n - len(b))
        one = Staged(ctx, [b])
        ms = device_ms(one, c, reps=3)
        one.free()
        g = ctx.responses_translate_large(c, [b])[0]
        emit(what="serial_walk_worst_case", layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))
    ctx.close()


CARD = "unknown"
if __name__ == "__main__":
    CARD = card()
    main()
