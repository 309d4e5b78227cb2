"""Throughput and latency of aigw_messages_translate_large_* (/v1/messages to OpenAI chat completions and to AWS Bedrock Converse)
on the Anthropic-format agent transcripts of tests/test_messages_large_cpu.py: the device call (CUDA events, median of 10) on the
corpus and on the transcripts with a 1 MiB tool_use input, the single-request time at about 1 MiB, and the serial walk's worst
cases.  Prints one JSON line per measurement, each with the card's name and power limit read in the same run.  Needs an H100;
there is no CPU path."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import bench_chat_large as B  # noqa: E402

GPU_SCHEMA = {"openai": "msg-openai", "aws-bedrock": "msg-aws-bedrock"}


def emit(**kw):
    kw["card"] = B.CARD
    print(json.dumps(kw), flush=True)


def main():
    import aigw_b200 as A
    import test_messages_large_cpu as ML
    ctx = A.Context(0)
    corpus = ML.agent_corpus() + ML.big_input_corpus()
    dev = "messages_translate_large_device"
    for schema in ML.SCHEMAS:
        c = ctx.cfg(GPU_SCHEMA[schema])
        got = ctx.messages_translate_large(c, corpus)
        assert all(g["status"] == A.AIGW_OK for g in got), [(g["status"], g["reason"]) for g in got]
        ms, used = B.device_call(ctx, c, corpus, fn=dev)
        nbytes = sum(map(len, corpus))
        emit(what="device_call", target=schema, requests=len(corpus), request_bytes=nbytes, output_bytes=used, ms=round(ms, 3),
             mb_per_s_in=round(nbytes / ms / 1e3, 1), max_len=max(map(len, corpus)))
        # one request of about 1 MiB: the kernel time and the host call's wall time
        b = ML.agent_corpus()[3]
        ms1, _ = B.device_call(ctx, c, [b], fn=dev)
        arena, offs, lens = A.pack_bodies([b])
        ctx.messages_translate_large_host(c, arena, offs, lens)
        t = []
        for _ in range(10):
            t0 = time.perf_counter(); ctx.messages_translate_large_host(c, arena, offs, lens); t.append(time.perf_counter() - t0)
        emit(what="single_request", target=schema, bytes=len(b), kernel_ms=round(ms1, 3), wall_ms_p50=round(1e3 * float(np.median(t)), 2))
        # the 1 MiB tool_use input alone
        one = ML.big_input_corpus()[0]
        ms2, _ = B.device_call(ctx, c, [one], fn=dev)
        emit(what="single_request_big_input", target=schema, bytes=len(one), kernel_ms=round(ms2, 3))
    # serial worst cases: 16 MiB of one-word text blocks, and tool_use inputs at the key-order work budget
    n = (16 << 20) - 4096
    words = json.dumps({"model": "m", "max_tokens": 1, "messages": [{"role": "user", "content": [{"type": "text", "text": "x" * 14}] * (n // 40)}]},
                       separators=(",", ":")).encode()
    import test_messages_large_gpu as T
    keys = ["k%02d" % i for i in range(40)]
    m = T.BUDGET // T._visit_work([keys])
    while T._visit_work([keys] * m) > T.BUDGET:
        m -= 1
    blocks = [{"type": "tool_use", "id": "t%d" % i, "name": "f", "input": {k: "v" * 8 for k in keys}} for i in range(m)]
    work = json.dumps({"model": "m", "max_tokens": 1, "messages": [{"role": "user", "content": "hi"}, {"role": "assistant", "content": blocks}]},
                      separators=(",", ":")).encode()
    for schema in ML.SCHEMAS:
        c = ctx.cfg(GPU_SCHEMA[schema])
        for label, b in (("one_word_text_blocks", words), ("inputs_at_work_budget", work)):
            ms, _ = B.device_call(ctx, c, [b], reps=3, fn=dev)
            g = ctx.messages_translate_large(c, [b])[0]
            emit(what="serial_walk_worst_case", target=schema, layout=label, bytes=len(b), ms=round(ms, 1), status=int(g["status"]), reason=int(g["reason"]))
    ctx.close()


if __name__ == "__main__":
    B.CARD = B.card()
    main()
