#!/usr/bin/env python3
"""Measurement of the /v1/responses response path: N streams x M ResponseBody calls of realistic Responses API events through
aigw_stream_chunks_soa (stream kind openai-responses, each call one event block), and buffered openai.Response bodies through
aigw_responses_response_usage_device.  Prints one JSON line with calls/s, bodies/s and bytes/s, the card's name and power limit,
and a CPU leg: the Python oracle (tests/_responses_oracle.py) on a sample, single-threaded."""
import argparse, ctypes as C, json, os, random, subprocess, sys, time
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import _responses_oracle as R
import aigw_b200 as A
from aigw_b200 import capi

ap = argparse.ArgumentParser()
ap.add_argument("--streams", type=int, default=20_000)
ap.add_argument("--calls", type=int, default=16, help="ResponseBody calls per stream")
ap.add_argument("--bodies", type=int, default=200_000)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--cpu-sample", type=int, default=2000)
a = ap.parse_args()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power = [x.strip() for x in q.splitlines()[0].split(",")]
    return name, power


def response(i, usage):
    return {"id": "resp_%d" % i, "object": "response", "created_at": 1741290958, "status": "completed", "error": None, "incomplete_details": None,
            "instructions": "You are a helpful assistant.", "max_output_tokens": None, "model": "gpt-4.1-2025-04-14",
            "output": [{"id": "msg_%d" % i, "type": "message", "status": "completed", "role": "assistant",
                        "content": [{"type": "output_text", "text": "This is a test. " * 8, "annotations": []}]}] if usage else [],
            "parallel_tool_calls": True, "previous_response_id": None, "reasoning": {"effort": None, "summary": None}, "store": True, "temperature": 1.0,
            "text": {"format": {"type": "text"}}, "tool_choice": "auto", "tools": [], "top_p": 1.0, "truncation": "disabled", "user": None, "metadata": {},
            "usage": {"input_tokens": 12 + i % 7, "input_tokens_details": {"cached_tokens": 0}, "output_tokens": 40, "output_tokens_details": {"reasoning_tokens": 0},
                      "total_tokens": 52 + i % 7} if usage else None}


def calls_of(i, m):
    """m event blocks: response.created, m-2 output_text deltas, response.completed"""
    evs = [{"type": "response.created", "sequence_number": 0, "response": response(i, False)}]
    evs += [{"type": "response.output_text.delta", "sequence_number": k + 1, "item_id": "msg_%d" % i, "output_index": 0, "content_index": 0, "delta": " token"} for k in range(m - 2)]
    evs.append({"type": "response.completed", "sequence_number": m, "response": response(i, True)})
    return [("event: %s\ndata: %s\n\n" % (e["type"], json.dumps(e, separators=(",", ":")))).encode() for e in evs]


name, power = card()
ctx = A.Context(0)
rng = random.Random(3)
# ---- stream leg: call k of every stream is one batch
per = [calls_of(i, a.calls) for i in range(a.streams)]
rounds = []
for k in range(a.calls):
    blob = b"".join(p[k] for p in per)
    pin, _ = ctx.host_array(len(blob) + 64); pin[:len(blob)] = np.frombuffer(blob, dtype=np.uint8)
    lens = np.array([len(p[k]) for p in per], dtype=np.uint32)
    offs = np.zeros(a.streams, dtype=np.uint64); offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    rounds.append((pin, offs, lens))
stream_bytes = sum(int(r[2].sum()) for r in rounds)


def stream_pass():
    hs = np.array(ctx.stream_open("openai-responses", b"gpt-4.1", n=a.streams), dtype=np.uint64)
    res = None
    for pin, offs, lens in rounds:
        res, _ = ctx.stream_chunks_soa(hs, pin, offs, lens, res=res)
    ctx.stream_close(list(hs))
    return res


for _ in range(a.warmup): stream_pass()
t = time.perf_counter()
for _ in range(a.steps): res = stream_pass()
s_wall = (time.perf_counter() - t) / a.steps
assert (res["status"] == 0).all() and (res["mask"] == 63).all() and (res["input"] == np.array([12 + i % 7 for i in range(a.streams)])).all()
# ---- buffered leg, device-resident
bodies = [json.dumps(response(i, True), separators=(",", ":")).encode() for i in range(a.bodies)]
arena, offs, lens = A.pack_bodies(bodies)
L, h = ctx.L, ctx.h
d_b, d_o, d_l, d_r = (L.aigw_device_alloc(h, max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, a.bodies * capi.SseResult.itemsize))
for d, x in ((d_b, arena), (d_o, offs), (d_l, lens)):
    assert L.aigw_memcpy_h2d(h, d, x.ctypes.data, x.nbytes) == 0
ms = C.c_float(0)
for _ in range(a.warmup): assert L.aigw_responses_response_usage_device(h, d_b, d_o, d_l, a.bodies, d_r, None, C.byref(ms)) == 0
kms = []
for _ in range(a.steps):
    assert L.aigw_responses_response_usage_device(h, d_b, d_o, d_l, a.bodies, d_r, None, C.byref(ms)) == 0
    kms.append(ms.value)
out = np.zeros(a.bodies, dtype=capi.SseResult)
assert L.aigw_memcpy_d2h(h, out.ctypes.data, d_r, out.nbytes) == 0
assert (out["status"] == 0).all() and (out["mask"] == 63).all()
for d in (d_b, d_o, d_l, d_r): L.aigw_device_free(h, d)
b_s = float(np.mean(kms)) / 1e3
body_bytes = int(lens.sum())
# ---- CPU leg: the oracle on a sample
ns = min(a.cpu_sample, a.streams)
t = time.perf_counter()
for i in range(ns):
    o = R.ResponsesSSEStream(b"gpt-4.1")
    for c in per[i]: o.feed(c)
cpu_calls = ns * a.calls / (time.perf_counter() - t)
nb = min(a.cpu_sample, a.bodies)
t = time.perf_counter()
for b in bodies[:nb]: R.response_responses(b)
cpu_bodies = nb / (time.perf_counter() - t)
print(json.dumps({"metric": "/v1/responses response path", "gpu": name, "power_limit": power,
                  "stream": {"streams": a.streams, "calls_per_stream": a.calls, "calls_per_s": a.streams * a.calls / s_wall, "bytes_per_s": stream_bytes / s_wall,
                             "timing": "host wall clock over whole passes (open, one aigw_stream_chunks_soa call per round from mapped pinned memory, close)"},
                  "buffered": {"bodies": a.bodies, "bodies_per_s": a.bodies / b_s, "bytes_per_s": body_bytes / b_s, "mean_body_bytes": body_bytes / a.bodies,
                               "timing": "CUDA events around the kernel (kernel_ms), device-resident bodies"},
                  "cpu_oracle": {"calls_per_s": cpu_calls, "bodies_per_s": cpu_bodies, "threads": 1, "kind": "Python restatement, not the Go reference"}}))
