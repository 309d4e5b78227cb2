"""GPU parity for the response side of /v1/responses (internal/translator/openai_responses.go:102-192): the stream usage scan as
stream kind 'openai-responses' (one ResponseBody call per chunk, no carry between calls) and the buffered branch
(aigw_responses_response_usage_*), against the reference's answers (tests/golden/responses_cases.json, the data-plane goldens) and
the oracle (tests/_responses_oracle.py) on seeded corpora under random chunkings."""
import json
import os
import random

import numpy as np
import pytest

import _responses_oracle as R

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "responses_cases.json"), encoding="utf-8"))
UPSTREAM = {c["name"]: c for c in json.load(open(os.path.join(HERE, "golden", "testupstream_cases.json"), encoding="utf-8"))["cases"]}
OKS, INTERNAL, DECLINED = 0, 3, 4
UNCHANGED = 0


@pytest.fixture(scope="module")
def gw():
    from aigw_b200 import capi
    g = capi.Context(0)
    yield g
    g.close()


def _events(data):
    """the stream cut after every event (blank line)"""
    parts, pos = [], 0
    while True:
        j = data.find(b"\n\n", pos)
        if j < 0:
            break
        parts.append(data[pos:j + 2]); pos = j + 2
    if pos < len(data):
        parts.append(data[pos:])
    return parts


def test_stream_reference_vectors_feed_by_feed(gw):
    streams = [(s["name"], s["data"].encode(), s["request_model"].encode()) for s in GOLD["streams"]]
    streams.append(("data-plane stream", UPSTREAM["openai - /v1/responses - stream"]["responseBody"].encode(), b"something"))
    for name, data, req in streams:
        (h,) = gw.stream_open("openai-responses", req)
        orc = R.ResponsesSSEStream(req)
        seen = []
        for feed in _events(data):
            r = gw.stream_chunk(h, feed, False)
            v, u = orc.feed(feed)
            assert v == R.OK and r["status"] == OKS and r["body_kind"] == UNCHANGED and r["body"] == b"", name
            assert r["usage"] == u.as_tuple(), name
            assert r["model"] == orc.model(), name
            assert r["carry_len"] == 0, name
            if u.mask:
                seen.append(r["usage"])
        gw.stream_close([h])
        exp = next((s["exp"] for s in GOLD["streams"] if s["name"] == name), "any")
        if exp == [-1] * 6:
            assert seen == [], name
        elif exp not in ("any", None):
            assert [[x[0], x[3], x[4], x[1], x[2], x[5]] for x in seen] == [exp], name
    assert GOLD["streams"][0]["exp"] == [10, 5, 15, 2, 0, 0]


def test_stream_one_byte_per_call(gw):
    """no line is ever whole within one call: no usage, the request model throughout, no carry"""
    data = GOLD["streams"][0]["data"].encode()
    (h,) = gw.stream_open("openai-responses", b"req-model")
    for i in range(len(data)):
        r = gw.stream_chunk(h, data[i:i + 1], False)
        assert r["status"] == OKS and r["usage"] == (-1,) * 6 and r["model"] == b"req-model" and r["carry_len"] == 0, i
    gw.stream_close([h])


def test_large_completed_event(gw):
    """a response.completed of ~60 KB in one call: above the 15.6 KB carry of the other kinds, processed in place"""
    text = "x" * 60000
    ev = {"type": "response.completed", "sequence_number": 9, "response": {"id": "r", "object": "response", "created_at": 1, "model": "m", "status": "completed",
          "output": [{"type": "message", "id": "m1", "status": "completed", "role": "assistant", "content": [{"type": "output_text", "text": text, "annotations": []}]}],
          "usage": {"input_tokens": 7, "input_tokens_details": {"cached_tokens": 1}, "output_tokens": 9, "output_tokens_details": {"reasoning_tokens": 2}, "total_tokens": 16}}}
    (h,) = gw.stream_open("openai-responses", b"req")
    r = gw.stream_chunk(h, ("data: " + json.dumps(ev) + "\n\n").encode(), False)
    assert r["status"] == OKS and r["usage"] == (7, 1, 0, 9, 16, 2) and r["carry_len"] == 0
    gw.stream_close([h])


# ---- seeded corpus: shapes as real OpenAI events carry them, plus perturbations
def _response(rng, model, usage, realistic):
    out = []
    for _ in range(rng.randint(0, 3)):
        k = rng.random()
        if k < 0.5:
            part = {"type": "output_text", "text": rng.choice(["Hello", "naïve 中文", "tab\tnew\nline", ""]), "annotations": []}
            if rng.random() < 0.3:
                part["annotations"] = [{"type": "url_citation", "start_index": 0, "end_index": 5, "url": "https://e.x", "title": "t"},
                                       {"type": "file_citation", "file_id": "f", "filename": "a.txt", "index": 1}][:rng.randint(1, 2)]
            if rng.random() < 0.2:
                part["logprobs"] = [{"token": "He", "bytes": [72, 101], "logprob": -0.1, "top_logprobs": [{"token": "he", "bytes": [104], "logprob": -2.5}]}]
            content = [part] if rng.random() < 0.9 else [{"type": "refusal", "refusal": "no"}]
            out.append({"id": "msg_1", "type": "message", "status": "completed", "role": "assistant", "content": content})
        elif k < 0.75:
            out.append({"type": "function_call", "id": "fc_1", "call_id": "call_1", "name": "get_weather", "arguments": "{\"city\":\"Paris\"}", "status": "completed"})
        else:
            out.append({"type": "reasoning", "id": "rs_1", "summary": [{"type": "summary_text", "text": "thinking"}], "encrypted_content": "gAAAA", "status": None})
    r = {"id": "resp_1", "object": "response", "created_at": 1741290958, "status": "completed", "error": None, "incomplete_details": None,
         "instructions": rng.choice([None, "You are a helpful assistant."]), "max_output_tokens": None, "model": model, "output": out,
         "parallel_tool_calls": True, "previous_response_id": None, "reasoning": {"effort": rng.choice([None, "low"]), "summary": None}, "store": True,
         "temperature": 1.0, "text": {"format": rng.choice([{"type": "text"}, {"type": "json_object"},
                                                           {"type": "json_schema", "name": "s", "schema": {"type": "object"}, "strict": True}]), "verbosity": "medium"},
         "tool_choice": rng.choice(["auto", "none", {"type": "function", "name": "get_weather"}]),
         "tools": rng.choice([[], [{"type": "function", "name": "get_weather", "description": "d", "parameters": {"type": "object", "properties": {}}, "strict": True}]]),
         "top_p": 1.0, "truncation": "disabled", "usage": usage, "user": None, "metadata": rng.choice([{}, {"k": "v"}])}
    if rng.random() < 0.3:
        r["conversation"] = {"id": "conv_1"}
        r["prompt"] = {"id": "pmpt_1", "version": "2"}
        r["completed_at"] = rng.choice([None, 1741290960])
    if not realistic:
        roll = rng.random()
        if roll < 0.15:
            r["output"].append({"type": rng.choice(["mcp_call", "web_search_call", "compaction"]), "id": "x"})        # known, not restated
        elif roll < 0.25:
            r["output"].append({"type": "no_such_item", "id": "x"})                                               # unknown tag: decode error
        elif roll < 0.35:
            r["output"].append({"type": "message", "role": 5, "content": []})                                     # type error deep inside
        elif roll < 0.42:
            r["tools"] = [{"type": "web_search"}]
        elif roll < 0.48:
            r["instructions"] = [{"type": "message", "role": "system", "content": "x"}]
        elif roll < 0.54:
            r["created_at"] = rng.choice([None, "1", 1.5])
        elif roll < 0.60:
            r["output"].append({"type": "message", "content": None})
        elif roll < 0.65:
            r["tool_choice"] = {"type": "mcp", "server_label": "s"}
    return r


def _usage(rng):
    u = {"input_tokens": rng.randint(0, 5000), "output_tokens": rng.randint(0, 3000)}
    u["total_tokens"] = u["input_tokens"] + u["output_tokens"]
    if rng.random() < 0.8:
        u["input_tokens_details"] = {"cached_tokens": rng.randint(0, 99)}
        if rng.random() < 0.3:
            u["input_tokens_details"]["cache_creation_input_tokens"] = rng.randint(0, 9)
    if rng.random() < 0.8:
        u["output_tokens_details"] = {"reasoning_tokens": rng.randint(0, 500)}
    if rng.random() < 0.05:
        u["total_tokens"] = rng.choice([4294967299, -3, "12"])
    return u


def _stream(rng, realistic):
    model = rng.choice(["gpt-4o-2024-11-20", "o3-mini", ""])
    evs = [{"type": "response.created", "sequence_number": 0, "response": _response(rng, model, None, realistic)},
           {"type": "response.in_progress", "sequence_number": 1, "response": _response(rng, model, None, realistic)},
           {"type": "response.output_item.added", "output_index": 0, "item": {"id": "msg_1", "type": "message", "status": "in_progress", "role": "assistant", "content": []}}]
    for k in range(rng.randint(0, 6)):
        evs.append({"type": "response.output_text.delta", "item_id": "msg_1", "output_index": 0, "content_index": 0, "delta": "tok%d" % k})
    resp = _response(rng, model, _usage(rng), realistic)
    if rng.random() < 0.1:   # a large completed event
        resp["output"].append({"type": "message", "id": "m", "role": "assistant", "content": [{"type": "output_text", "text": "y" * rng.randint(48000, 60000), "annotations": []}]})
    evs.append({"type": "response.completed", "sequence_number": 99, "response": resp})
    lines = []
    for e in evs:
        if not realistic and rng.random() < 0.04:
            lines.append(rng.choice(["data: {invalid json}", "data: [DONE]", ": keep-alive", "data: ", "data: null", "data: {\"type\":5}"]))
        lines.append("event: " + e["type"])
        lines.append("data: " + json.dumps(e, separators=rng.choice([(",", ":"), (", ", ": ")]), ensure_ascii=rng.random() < 0.5))
        lines.append("")
    return ("\n".join(lines) + "\n").encode()


def _chunk(rng, data):
    roll = rng.random()
    if roll < 0.4:
        return _events(data)                                         # event aligned
    cuts = sorted(set(rng.sample(range(1, len(data)), min(rng.randint(1, 8), len(data) - 1))))
    return [data[a:b] for a, b in zip([0] + cuts, cuts + [len(data)])]   # split lines


def _run_corpus(gw, streams):
    n = len(streams)
    hs = gw.stream_open("openai-responses", b"req-model", n=n)
    orc = [R.ResponsesSSEStream(b"req-model") for _ in range(n)]
    dead = set()
    declined_in = set()
    with_usage = 0
    for rnd in range(max(len(s) for s in streams)):
        idx = [i for i in range(n) if rnd < len(streams[i]) and i not in dead]
        got = gw.stream_chunks([hs[i] for i in idx], [streams[i][rnd] for i in idx], [False] * len(idx))
        for i, g in zip(idx, got):
            v, u = orc[i].feed(streams[i][rnd])
            if g["status"] == DECLINED:
                assert v == R.OUT, (i, rnd, streams[i][rnd][:300])   # every decline is an input outside the restated subset
                dead.add(i); declined_in.add(i); continue
            if v == R.OUT:   # the GPU went on: its answer is not checked, the stream is no longer followed
                dead.add(i); continue
            assert g["status"] == OKS and g["carry_len"] == 0
            assert g["usage"] == u.as_tuple(), (i, rnd, streams[i][rnd][:300])
            assert g["model"] == orc[i].model(), (i, rnd)
            with_usage += 1 if u.mask else 0
    gw.stream_close(hs)
    return declined_in, with_usage


def test_stream_corpus_random_chunking_vs_oracle(gw):
    rng = random.Random(11)
    mixed = [_chunk(rng, _stream(rng, False)) for _ in range(160)]
    realistic = [_chunk(rng, _stream(rng, True)) for _ in range(96)]
    declined, with_usage = _run_corpus(gw, mixed + realistic)
    assert not [i for i in declined if i >= len(mixed)], "the realistic sub-corpus must not decline"
    print("responses stream corpus: declined", len(declined), "calls with usage", with_usage)
    assert with_usage > 60 and len(declined) > 0


def test_stream_completed_without_usage_declines(gw):
    for ev in (b'{"type":"response.completed","response":null}', b'{"type":"response.completed","response":{"usage":null}}',
               b'{"type":"response.completed","sequence_number":3}', b'{"type":"response.completed","response":{"id":"r","model":"m"}}'):
        (h,) = gw.stream_open("openai-responses", b"req")
        r = gw.stream_chunk(h, b"data: " + ev + b"\n\n", False)
        assert r["status"] == DECLINED, ev
        gw.stream_close([h])


def _unpack(r):
    m = int(r["mask"])
    return (int(r["input"]) if m & 1 else -1, int(r["output"]) if m & 2 else -1, int(r["total"]) if m & 4 else -1,
            int(r["cached"]) if m & 8 else -1, int(r["cache_creation"]) if m & 16 else -1, int(r["reasoning"]) if m & 32 else -1)


def _expect(u):
    return (u.input, u.output, u.total, u.cached, u.cache_creation, u.reasoning) if u.mask == 63 else (-1,) * 6


def _bodies():
    rng = random.Random(5)
    bodies = [c["body"].encode() for c in GOLD["buffered"]] + [UPSTREAM["openai - /v1/responses"]["responseBody"].encode()]
    for i in range(2600):
        realistic = rng.random() < 0.5
        b = json.dumps(_response(rng, rng.choice(["gpt-4o", "o3", ""]), rng.choice([_usage(rng), _usage(rng), None]), realistic),
                       separators=rng.choice([(",", ":"), (", ", ": ")]), ensure_ascii=rng.random() < 0.5).encode()
        roll = rng.random()
        if roll < 0.05 and len(b) > 2: b = b[: rng.randint(1, len(b) - 1)]                              # truncated
        elif roll < 0.10: b = b + rng.choice([b" ", b"\n\t", b" x", b"{}", b"]"])                      # trailing bytes are ignored
        elif roll < 0.13: b = b.replace(b'"input_tokens":', b'"input_tokens":4294967296', 1).replace(b'"input_tokens": ', b'"input_tokens": 4294967296', 1)
        elif roll < 0.15: b = b.replace(b'"usage":', b'"usage":[],"x":', 1).replace(b'"usage": ', b'"usage": [], "x": ', 1)
        bodies.append(b)
    bodies += [b"null", b"[]", b"{}", b'{"usage":null,"model":"m"}', b'{"usage":{}}', b"", b"  ", b'{"model":"a\\u0062"}', b'{"mod\\u0065l":"x"}',
               b'{"usage":{"input_tokens":-1,"output_tokens":9223372036854775807}}', b'{"usage":{"input_tokens":9223372036854775808}}', b"{invalid json"]
    return bodies


def _check_buffered(res, raw, bodies, costs=None):
    n_ok = n_decl = n_err = 0
    for i, b in enumerate(bodies):
        v, u, model = R.response_responses(b)
        r = res[i]
        if int(r["status"]) == DECLINED:
            assert v == R.OUT, (i, b[:300]); n_decl += 1; continue
        if v == R.OUT:
            continue
        if v == R.FAIL:
            assert int(r["status"]) == INTERNAL, (i, b[:200]); n_err += 1; continue
        assert int(r["status"]) == OKS, (i, b[:200])
        assert _unpack(r) == _expect(u), (i, b[:300])
        assert raw[int(r["model_off"]):int(r["model_off"]) + int(r["model_len"])] == model, (i, b[:200])
        if costs is not None:
            e = _expect(u)
            assert [int(x) for x in costs[i]] == [max(e[0], 0), max(e[3], 0), max(e[4], 0), max(e[1], 0), max(e[2], 0), max(e[5], 0)], i
        n_ok += 1
    return n_ok, n_err, n_decl


def test_buffered_reference_vectors(gw):
    import aigw_b200 as A
    bodies = [c["body"].encode() for c in GOLD["buffered"]]
    arena, offs, lens = A.pack_bodies(bodies)
    res, _ = gw.response_usage_host(arena, offs, lens, responses=True)
    raw = bytes(arena)
    for c, r in zip(GOLD["buffered"], res):
        if c["exp_error"]:
            assert int(r["status"]) == INTERNAL, c["name"]
            continue
        assert int(r["status"]) == OKS and list(_unpack(r)) == c["exp"], c["name"]
        assert raw[int(r["model_off"]):int(r["model_off"]) + int(r["model_len"])].decode() == c["exp_model"], c["name"]


def test_buffered_corpus_vs_oracle_host(gw):
    import aigw_b200 as A
    bodies = _bodies()
    arena, offs, lens = A.pack_bodies(bodies)
    res, costs = gw.response_usage_host(arena, offs, lens, cost_types=(0, 1, 2, 3, 4, 5), responses=True)
    n_ok, n_err, n_decl = _check_buffered(res, bytes(arena), bodies, costs)
    print("responses buffered: ok", n_ok, "errors", n_err, "declined", n_decl)
    assert n_ok > 1500 and n_err > 100 and n_decl > 50


def test_buffered_corpus_vs_oracle_device(gw):
    import ctypes as C
    import aigw_b200 as A
    from aigw_b200 import capi
    bodies = _bodies()
    arena, offs, lens = A.pack_bodies(bodies)
    n = len(bodies)
    L, h = gw.L, gw.h
    d_b, d_o, d_l, d_r = (L.aigw_device_alloc(h, max(16, x)) for x in (arena.nbytes, offs.nbytes, lens.nbytes, n * capi.SseResult.itemsize))
    try:
        for d, a in ((d_b, arena), (d_o, offs), (d_l, lens)):
            assert L.aigw_memcpy_h2d(h, d, a.ctypes.data, a.nbytes) == 0
        ms = C.c_float(0)
        assert L.aigw_responses_response_usage_device(h, d_b, d_o, d_l, n, d_r, None, C.byref(ms)) == 0
        assert L.aigw_sync(h) == 0
        res = np.zeros(n, dtype=capi.SseResult)
        assert L.aigw_memcpy_d2h(h, res.ctypes.data, d_r, res.nbytes) == 0
    finally:
        for d in (d_b, d_o, d_l, d_r):
            L.aigw_device_free(h, d)
    n_ok, n_err, n_decl = _check_buffered(res, bytes(arena), bodies)
    assert n_ok > 1500 and n_err > 100
