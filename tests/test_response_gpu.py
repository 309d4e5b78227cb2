"""GPU parity for non-stream OpenAI-schema responses (R1) and the direct cost selectors (C2)."""
import json
import os
import random

import numpy as np
import pytest

import _oracle as O

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def _bodies(seed, n):
    r = random.Random(seed)
    out = []
    for i in range(n):
        usage = {"prompt_tokens": r.randint(0, 5000), "completion_tokens": r.randint(0, 3000)}
        usage["total_tokens"] = usage["prompt_tokens"] + usage["completion_tokens"]
        if r.random() < 0.5:
            usage["prompt_tokens_details"] = {"cached_tokens": r.randint(0, 100), "audio_tokens": 0}
            if r.random() < 0.3:
                usage["prompt_tokens_details"]["cache_creation_input_tokens"] = r.randint(0, 50)
        if r.random() < 0.4:
            usage["completion_tokens_details"] = {"reasoning_tokens": r.randint(0, 900), "audio_tokens": 0, "accepted_prediction_tokens": 0, "rejected_prediction_tokens": 0}
        msg = {"role": "assistant", "content": "answer " * r.randint(1, 80), "refusal": None}
        if r.random() < 0.2:
            msg["tool_calls"] = [{"id": "call_1", "type": "function", "function": {"name": "f", "arguments": "{\"a\":1}"}}]
            msg["content"] = None
        if r.random() < 0.1:
            msg["annotations"] = [{"type": "url_citation", "url_citation": {"end_index": 5, "start_index": 1, "url": "https://x", "title": "t"}}]
        if r.random() < 0.1:
            msg["reasoning_content"] = r.choice(["thinking...", {"reasoningContent": {"reasoningText": {"text": "t", "signature": "c2ln"}}}])
        d = {"id": "chatcmpl-%d" % i, "object": "chat.completion", "created": 1731618222, "model": r.choice(["gpt-4o-mini-2024-07-18", "gpt-4o", ""]),
             "choices": [{"index": 0, "message": msg, "logprobs": None, "finish_reason": "stop"}], "usage": usage, "system_fingerprint": "fp_x"}
        if r.random() < 0.1:
            del d["usage"]
        if r.random() < 0.1:
            del d["model"]
        sep = r.choice([(",", ":"), (", ", ": ")])
        b = json.dumps(d, separators=sep).encode()
        roll = r.random()
        if roll < 0.04: b = b[: r.randint(1, len(b) - 1)]                                  # truncated
        elif roll < 0.07: b = b.replace(b'"prompt_tokens":', b'"prompt_tokens":"x",  "zz":', 1)   # still valid, extra key
        elif roll < 0.10: b = b.replace(b'"index":0', b'"index":"0"', 1).replace(b'"index": 0', b'"index": "0"', 1)   # type error
        elif roll < 0.13: b = b.replace(b'"created":1731618222', b'"created":1731618222.75', 1).replace(b'"created": 1731618222', b'"created": 1.5e3', 1)
        elif roll < 0.16: b = b + b"  trailing garbage"
        elif roll < 0.18: b = b.replace(b'"total_tokens"', b'"total_tokens":4294967299,"x"', 1)
        out.append(b)
    out += [b"null", b"[]", b"{}", b'{"usage":null,"model":"m"}', b'{"usage":{"total_tokens":7.5}}', b'{"choices":null}', b"", b"   ", b'{"model":"a\\u0062"}', b'{"mod\\u0065l":"x"}']
    return out


def test_response_usage_parity(ctx):
    import aigw_b200 as A
    bodies = _bodies(7, 3000)
    arena, offs, lens = A.pack_bodies(bodies)
    res, costs = ctx.response_usage_host(arena, offs, lens, cost_types=(0, 1, 2, 3, 4, 5))
    raw = bytes(arena)
    n_ok = 0
    for i, b in enumerate(bodies):
        ok, u, model = O.response_openai(b, b"")
        r = res[i]
        if int(r["status"]) == A.AIGW_DECLINED:
            continue
        if not ok:
            assert int(r["status"]) == A.AIGW_INTERNAL, (i, b[:200])
            continue
        assert int(r["status"]) == 0, (i, b[:200])
        n_ok += 1
        m = int(r["mask"])
        got = (int(r["input"]) if m & 1 else -1, int(r["cached"]) if m & 8 else -1, int(r["cache_creation"]) if m & 16 else -1,
               int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1, int(r["reasoning"]) if m & 32 else -1)
        assert got == u.as_tuple(), (i, b[:300], got, u.as_tuple())
        assert raw[int(r["model_off"]):int(r["model_off"]) + int(r["model_len"])] == model
        for k in range(6):
            assert int(costs[i, k]) == O.eval_cost(k, u)
    assert n_ok > 2400


def test_response_usage_host_any_offset_order(ctx):
    """the host form stages every body whatever the order of the offset table: with the last two rows of the offset and length
    tables swapped, each record equals the record of the same body in arena order"""
    import aigw_b200 as A
    bodies = [json.dumps({"id": "chatcmpl-%d" % i, "object": "chat.completion", "model": "gpt-4o-mini",
                          "choices": [{"index": 0, "message": {"role": "assistant", "content": "ok " * (i % 9)}, "finish_reason": "stop"}],
                          "usage": {"prompt_tokens": i, "completion_tokens": 2 * i, "total_tokens": 3 * i}}, separators=(",", ":")).encode() for i in range(300)]
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    perm = np.arange(n)
    perm[[n - 2, n - 1]] = perm[[n - 1, n - 2]]
    # the swapped call runs first, so that no earlier call of this test has staged the last body's bytes
    swapped, swapped_costs = ctx.response_usage_host(arena, offs[:n][perm].copy(), lens[perm].copy(), cost_types=(0, 3, 4))
    ordered, costs = ctx.response_usage_host(arena, offs, lens, cost_types=(0, 3, 4))
    assert (ordered["status"] == 0).all() and int(ordered[n - 1]["input"]) == n - 1
    assert ordered[perm].tobytes() == swapped.tobytes()
    assert np.array_equal(costs[perm], swapped_costs)


def test_reference_response_golden(ctx):
    """testupstream_test.go:266: OpenAI passthrough response without usage: counters set to zero, no model."""
    import aigw_b200 as A
    b = b'{"choices":[{"message":{"content":"This is a test."}}]}'
    arena, offs, lens = A.pack_bodies([b])
    res, _ = ctx.response_usage_host(arena, offs, lens)
    r = res[0]
    assert int(r["status"]) == 0 and int(r["mask"]) == 7 and (int(r["input"]), int(r["output"]), int(r["total"])) == (0, 0, 0) and int(r["model_len"]) == 0


def test_embeddings_response_usage_parity(ctx):
    """R1 for /v1/embeddings (internal/translator/openai_embeddings.go:70-88): usage (input + total only) and response model."""
    import json as _json
    from aigw_b200 import capi
    rng = np.random.default_rng(4)
    bodies = []
    for i in range(600):
        n = int(rng.integers(0, 6))
        data = [{"object": "embedding", "index": k, "embedding": ([float(x) for x in np.round(rng.normal(size=int(rng.integers(1, 200))), 6)] if rng.integers(0, 3) else "AAECAwQF")} for k in range(n)]
        d = {"object": "list", "data": data, "model": ["text-embedding-3-small", "text-embedding-ada-002", ""][int(rng.integers(0, 3))],
             "usage": {"prompt_tokens": int(rng.integers(0, 9000)), "total_tokens": int(rng.integers(0, 9000))}}
        if i % 11 == 0: del d["usage"]
        if i % 13 == 0: d["model"] = None
        bodies.append(_json.dumps(d, separators=(",", ":")).encode())
    bodies += [b'{"data":[{"embedding":{"a":1}}]}', b'{"data":[{"embedding":[1,"x"]}]}', b'{"usage":{"prompt_tokens":1.5}}', b'{"data":[{"embedding":null},null],"usage":null}', b'null', b'[]', b'{"model":5}',
               b'{"data":[{"embedding":[1e-3,-2.5E+2,0]}],"usage":{"prompt_tokens":4294967297,"total_tokens":3}}']
    arena, offs, lens = capi.pack_bodies(bodies)
    res, _ = ctx.response_usage_host(arena, offs, lens, embeddings=True)
    for b, r, o in zip(bodies, res, offs):
        ok, u, m = O.response_embeddings(b)
        if r["status"] == 4:
            continue
        assert (r["status"] == 0) == ok, (b[:120], int(r["status"]), ok)
        if ok:
            assert (int(r["input"]), int(r["output"]), int(r["total"]), int(r["mask"])) == (u.input, 0, u.total, 5), b[:120]
            got = bytes(arena[int(r["model_off"]):int(r["model_off"]) + int(r["model_len"])])
            assert got == m
    assert (res["status"] != 4).sum() >= len(bodies) - 2
