"""Throughput and latency of aigw_chat_translate_large_* and aigw_chat_bedrock_translate_large_* on the long agent transcripts of
tests/test_chat_large_cpu.py: the device call and the host call end to end (OpenAI with the model override and forced
include_usage, Azure, and AWS Bedrock with and without an override, also on the transcripts re-serialised with ensure_ascii),
single-request wall latency at 128 KiB, 1 MiB and 4 MiB, and the serial walk's worst cases.  Prints one JSON line per measurement, each with the card's
name and power limit read in the same run.  Needs an H100; there is no CPU path."""
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


def device_call(ctx, c, bodies, reps=10, fn="chat_translate_large_device"):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    cap = sum(3 * len(b) + 1024 for b in bodies)
    d_b, d_o, d_l, d_out, d_r, d_u = (ctx.dalloc(max(16, x)) for x in (arena.nbytes + 64, offs.nbytes, lens.nbytes, cap, n * 32, 8))
    try:
        ctx.h2d(d_b, arena); ctx.h2d(d_o, offs); ctx.h2d(d_l, lens)
        ms = []
        for i in range(reps + 2):
            ctx.memset(d_u, 0, 8)
            t = getattr(ctx, fn)(c, d_b, d_o, d_l, n, int(lens.max()), d_out, cap, d_r, d_u)
            if i >= 2:
                ms.append(t)
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, d_u)
        return float(np.median(ms)), int(used[0])
    finally:
        for d in (d_b, d_o, d_l, d_out, d_r, d_u):
            ctx.dfree(d)


def main():
    import aigw_b200 as A
    import test_chat_large_cpu as L
    ctx = A.Context(0)
    corpus = L.realistic_corpus()
    for name, schema, override in (("openai_override_usage", "openai", "gpt-4o-mini-2024"), ("azure", "azure-openai", None)):
        c = ctx.cfg(schema, model_override=override, cost_configured=True, api_version="2025-01-01-preview" if schema == "azure-openai" else None)
        got = ctx.chat_translate_large(c, corpus)
        assert all(g["status"] == A.AIGW_OK for g in got), [(g["status"], g["reason"]) for g in got]
        ms, used = device_call(ctx, c, corpus)
        nbytes = sum(map(len, corpus))
        emit(what="device_call", target=name, requests=len(corpus), request_bytes=nbytes, output_bytes=used, ms=round(ms, 3),
             gb_per_s_in=round(nbytes / ms / 1e6, 2), max_len=max(map(len, corpus)))
        arena, offs, lens = A.pack_bodies(corpus)
        ctx.chat_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.chat_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="host_call", target=name, ms=round(1e3 * float(np.median(t)), 2), gb_per_s_in=round(nbytes / float(np.median(t)) / 1e9, 2))
    # single requests: wall latency of one host call
    c = ctx.cfg("openai", model_override="gpt-4o-mini-2024", cost_configured=True)
    for size in (128 << 10, 1 << 20, 4 << 20):
        b = L.long_chat(77, size, "true")
        arena, offs, lens = A.pack_bodies([b])
        assert ctx.chat_translate_large(c, [b])[0]["status"] == A.AIGW_OK
        t = []
        for i in range(60):
            t0 = time.perf_counter(); ctx.chat_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        t = np.array(t[10:]) * 1e6
        ms, _ = device_call(ctx, c, [b], reps=10)
        emit(what="single_request_wall_us", bytes=len(b), p50=round(float(np.percentile(t, 50))), p99=round(float(np.percentile(t, 99))), kernel_ms=round(ms, 3))
    # the serial walk's worst case at 16 MiB - 1: every token in tool parameters (the key-sorting check of emit_any), or in
    # tool-call arguments (declined once their total passes 256 KiB), or an array of scalars in an ignored member (the grammar pass alone)
    n = (16 << 20) - 1
    obj = "{" + ",".join('"k%02d":11111' % i for i in range(60)) + "}"   # 5 tokens in 12 bytes: inside the token cap
    params = '{"model":"m","messages":[],"tools":[' + ",".join('{"type":"function","function":{"name":"f","parameters":%s}}' % obj for _ in range((n - 200) // (len(obj) + 60))) + "]}"
    args = json.dumps(json.loads(obj)).replace("\\", "\\\\").replace('"', '\\"')
    calls = '{"model":"m","messages":[{"role":"assistant","tool_calls":[' + ",".join('{"id":"a","function":{"name":"f","arguments":"%s"}}' % args for _ in range((n - 200) // (len(args) + 60))) + "]}]}"
    flat = '{"model":"m","x":[' + ",".join(["1111"] * ((n - 64) // 5)) + "]}"
    # 64 keys of about 260 KB that differ only in their last bytes: every compare of the key-order check reads a whole key
    longkeys = '{"model":"m","messages":[],"tools":[{"type":"function","function":{"name":"f","parameters":{' + ",".join(
        '"%s%02d":1' % ("k" * 260000, i) for i in range(64)) + "}}}]}"
    for label, s in (("tool_parameters", params), ("tool_parameters_long_keys", longkeys), ("tool_call_arguments", calls),
                     ("ignored_member_scalars", flat)):
        b = s.encode()
        b = b + b" " * (n - len(b))
        ms, _ = device_call(ctx, c, [b], reps=3)
        g = ctx.chat_translate_large(c, [b])[0]
        emit(what="serial_walk_worst_case", layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))
    bedrock(ctx, corpus)
    ctx.close()


def bedrock(ctx, corpus):
    import aigw_b200 as A
    import test_chat_bedrock_large_cpu as B
    import test_chat_large_cpu as L
    dev = "chat_bedrock_translate_large_device"
    dense = [json.dumps(json.loads(b), ensure_ascii=True).encode() for b in corpus]
    for name, bodies, override in (("bedrock", corpus, None), ("bedrock_override", corpus, "us.anthropic.claude-3-7-sonnet"), ("bedrock_ensure_ascii", dense, None)):
        c = ctx.cfg("aws-bedrock", model_override=override)
        got = ctx.chat_bedrock_translate_large(c, bodies)
        assert all(g["status"] == A.AIGW_OK for g in got), [(g["status"], g["reason"]) for g in got]
        ms, used = device_call(ctx, c, bodies, fn=dev)
        nbytes = sum(map(len, bodies))
        emit(what="device_call", target=name, requests=len(bodies), request_bytes=nbytes, output_bytes=used, ms=round(ms, 3),
             gb_per_s_in=round(nbytes / ms / 1e6, 2), max_len=max(map(len, bodies)))
        arena, offs, lens = A.pack_bodies(bodies)
        ctx.chat_bedrock_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(5):
            t0 = time.perf_counter(); ctx.chat_bedrock_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="host_call", target=name, ms=round(1e3 * float(np.median(t)), 2), gb_per_s_in=round(nbytes / float(np.median(t)) / 1e9, 2))
    c = ctx.cfg("aws-bedrock")
    for size in (128 << 10, 1 << 20, 4 << 20):
        b = L.long_chat(77, size, "true")
        arena, offs, lens = A.pack_bodies([b])
        assert ctx.chat_bedrock_translate_large(c, [b])[0]["status"] == A.AIGW_OK
        t = []
        for i in range(60):
            t0 = time.perf_counter(); ctx.chat_bedrock_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        t = np.array(t[10:]) * 1e6
        ms, _ = device_call(ctx, c, [b], reps=10, fn=dev)
        emit(what="single_request_wall_us", target="bedrock", bytes=len(b), p50=round(float(np.percentile(t, 50))), p99=round(float(np.percentile(t, 99))), kernel_ms=round(ms, 3))
    # the serial walk's worst cases of the shapes the Converse plan adds, at 16 MiB - 1: tiny user messages, one long run of tool
    # messages, and a string of re-spelled escapes
    n = (16 << 20) - 1
    tiny = '{"model":"m","messages":[' + ",".join(['{"role":"user","content":"hi"}'] * ((n - 64) // 31)) + "]}"
    tools = '{"model":"m","messages":[' + ",".join(['{"role":"tool","content":"r","tool_call_id":"i"}'] * ((n - 64) // 49)) + "]}"
    esc = '{"model":"m","messages":[{"role":"user","content":"' + "\\u00e9" * ((n - 64) // 6) + '"}]}'
    for label, s in (("tiny_user_messages", tiny), ("tool_message_run", tools), ("respelled_escapes", esc)):
        b = s.encode()
        b = b + b" " * (n - len(b))
        ms, _ = device_call(ctx, c, [b], reps=3, fn=dev)
        g = ctx.chat_bedrock_translate_large(c, [b])[0]
        emit(what="serial_walk_worst_case", target="bedrock", layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))


CARD = "unknown"
if __name__ == "__main__":
    CARD = card()
    main()
