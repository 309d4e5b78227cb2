"""The /v1/responses oracle (tests/_responses_oracle.py) against the reference's own answers: the translator tests
(openai_responses_test.go:517-811, lifted into tests/golden/responses_cases.json) and the data-plane goldens
"openai - /v1/responses" and "openai - /v1/responses - stream" (testupstream_test.go)."""
import importlib.util
import json
import os

import _responses_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "responses_cases.json"), encoding="utf-8"))
UPSTREAM = {c["name"]: c for c in json.load(open(os.path.join(HERE, "golden", "testupstream_cases.json"), encoding="utf-8"))["cases"]}


def _counters(u):
    return [u.input, u.output, u.total, u.cached, u.cache_creation, u.reasoning] if u.mask == 63 else [-1] * 6


def test_stream_reference_vectors():
    for s in GOLD["streams"]:
        o = R.ResponsesSSEStream(s["request_model"].encode())
        v, u = o.feed(s["data"].encode())
        assert v == R.OK, s["name"]
        if s["exp"] is not None:
            assert _counters(u) == s["exp"], s["name"]
        assert o.model().decode() == s["exp_model"], s["name"]


def test_buffered_reference_vectors():
    for c in GOLD["buffered"]:
        v, u, model = R.response_responses(c["body"].encode())
        if c["exp_error"]:
            assert v == R.FAIL, c["name"]
            continue
        assert v == R.OK, c["name"]
        assert _counters(u) == c["exp"] and model.decode() == c["exp_model"], c["name"]


def test_data_plane_goldens():
    c = UPSTREAM["openai - /v1/responses"]
    v, u, model = R.response_responses(c["responseBody"].encode())
    assert v == R.OK and model == b"something" and u.mask == 63
    c = UPSTREAM["openai - /v1/responses - stream"]
    o = R.ResponsesSSEStream(b"something")
    v, u = o.feed(c["responseBody"].encode())
    assert v == R.OK and u.mask == 63 and o.model().startswith(b"gpt-4.1-2")


def test_no_carry_between_calls():
    """a line cut across two calls is lost on both sides"""
    data = GOLD["streams"][0]["data"].encode()
    cut = data.index(b"response.completed") + 5
    o = R.ResponsesSSEStream(b"req")
    assert o.feed(data[:cut])[1].mask == 0
    assert o.feed(data[cut:])[1].mask == 0
    assert o.model() == b"gpt-4o-2024-11-20"


def test_decode_rules():
    ok = lambda b: R.response_responses(b)[0]
    assert ok(b"") == R.FAIL and ok(b"  ") == R.FAIL and ok(b"{invalid json") == R.FAIL
    assert ok(b'{"model":"m"} trailing') == R.OK and ok(b"null") == R.OK and ok(b"{}") == R.OK
    assert ok(b'{"instructions":null,"tool_choice":null,"completed_at":null}') == R.OK
    assert ok(b'{"created_at":null}') == R.FAIL and ok(b'{"output":[null]}') == R.FAIL
    assert ok(b'{"output":[{"type":"nope"}]}') == R.FAIL and ok(b'{"output":[{"type":"mcp_call"}]}') == R.OUT
    assert ok(b'{"output":[{"type":"message","content":null}]}') == R.FAIL
    assert ok(b'{"output":[{"type":"message","content":"hi"}]}') == R.OK
    assert ok(b'{"instructions":[]}') == R.OK and ok(b'{"instructions":[{"type":"message"}]}') == R.OUT
    assert ok(b'{"tool_choice":"auto"}') == R.OK and ok(b'{"tool_choice":{"type":"function","name":"f"}}') == R.OK
    assert ok(b'{"tool_choice":{"type":"mcp","server_label":"x"}}') == R.OUT and ok(b'{"tool_choice":{}}') == R.FAIL
    assert ok(b'{"presence_penalty":1e3}') == R.OUT and ok(b'{"presence_penalty":0.5}') == R.OK
    v, u, m = R.response_responses(b'{"usage":{"input_tokens":4294967297,"input_tokens_details":{"cache_creation_input_tokens":3}}}')
    assert v == R.OK and (u.input, u.cache_creation, u.mask) == (1, 3, 63)
    v, u, m = R.response_responses(b'{"usage":null,"model":"m"}')
    assert v == R.OK and u.mask == 0 and m == b"m"


def test_stream_panic_case_is_outside():
    for ev in (b'{"type":"response.completed","response":null}', b'{"type":"response.completed","response":{"usage":null}}', b'{"type":"response.completed"}'):
        assert R.ResponsesSSEStream().feed(b"data: " + ev + b"\n\n")[0] == R.OUT
    # a type error deep inside the event: the line is skipped
    v, u = R.ResponsesSSEStream().feed(b'data: {"type":"response.completed","response":{"usage":{"input_tokens":1},"output":[{"type":"message","role":5}]}}\n')
    assert v == R.OK and u.mask == 0


def test_host_build_of_the_step_matches_the_oracle():
    """the stream step compiled for the host (tools/stream_host_check.cpp) over the GPU test's seeded corpus"""
    spec = importlib.util.spec_from_file_location("stream_host_check", os.path.join(HERE, "..", "tools", "stream_host_check.py"))
    shc = importlib.util.module_from_spec(spec); spec.loader.exec_module(shc)
    with shc.Host() as H:
        declined, with_usage = shc.check_responses(H)
    assert declined > 0 and with_usage > 60
