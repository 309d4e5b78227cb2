"""Corpora of /v1/messages requests for aigw_messages_translate_large_* (test_messages_large_gpu.py feeds them through the GPU):
seeded Anthropic-format agent transcripts of 64 KiB to about 4 MiB in the subset the full re-maps accept (AIGW_SCHEMA_MSG_OPENAI,
AIGW_SCHEMA_MSG_AWS_BEDROCK): a large system prompt of text blocks (some with cache_control), 10 to 40 tools with nested
input_schema, every tool_choice form, assistant turns of text and several tool_use blocks with nested inputs (one of them a
multi-MiB file body), user turns of tool_result blocks with string, text-block and null content and is_error, stop_sequences,
top_k, float max_tokens, models that need PathEscape, and the ensure_ascii and indent re-serialisations.  Here: their shape, that
they are reproducible, the oracle's verdicts for both schemas with and without an override, and the densest records."""
import json

import numpy as np
import pytest

import _oracle as O
import test_chat_large_cpu as L

SCHEMAS = ("openai", "aws-bedrock")
PREFIX = "v1"
MODELS = ["claude-sonnet-4-5", "anthropic.claude-3-5-sonnet-20241022-v2:0", "arn:aws:bedrock:us-east-1:123456789012:inference-profile/us.anthropic.claude-3-7-sonnet",
          "claude opus 4"]
OVERRIDE = "us.anthropic.claude-sonnet-4-20250514-v1:0"
SIZES = (70_000, 150_000, 400_000, 1_200_000, 4_000_000)
TOOL_CHOICES = [None, {"type": "auto"}, {"type": "any"}, {"type": "none"}, {"type": "tool", "name": "tool_3"},
                {"type": "any", "disable_parallel_tool_use": True}, {"type": "auto", "disable_parallel_tool_use": None}]
CODE = ("def handler(request):\n    path = request.get(\"path\", \"/tmp/x\")\n    if not path.endswith(\"\\\\\"):\n"
        "        return {\"status\": 200, \"body\": open(path).read()}\n    raise ValueError('bad \"path\"')\n\n")


def oracle(schema, body, override=""):
    return O.messages_translate(schema, body, model_override=override, api_version=PREFIX if schema == "openai" else "")


def _file(rng, n):
    """a source file of about n bytes: code lines with quotes, backslashes, tabs and newlines, ASCII only (an input string with a
    \\u escape is outside both translators' subset)"""
    out, size = [], 0
    while size < n:
        if rng.random() < 0.5:
            out.append(CODE); size += len(CODE)
        else:
            s = "    # " + L._text(rng, int(rng.integers(20, 100)), escapes=False) + "\n"
            out.append(s); size += len(s)
    return "".join(out)[:n]


def _input(rng, big=0):
    """a nested tool_use input: a file write, an edit, a shell command or a search"""
    k = int(rng.integers(4))
    if big or k == 0:
        return {"file_path": "/work/src/mod_%d.py" % int(rng.integers(100)), "content": _file(rng, big or int(rng.integers(200, 4000))),
                "options": {"mode": "overwrite", "backup": bool(rng.random() < 0.5), "encoding": "utf-8"}}
    if k == 1:
        return {"file_path": "/work/README.md", "edits": [{"old_string": L._text(rng, 60, escapes=False), "new_string": _file(rng, 300),
                                                            "replace_all": False} for _ in range(int(rng.integers(1, 4)))]}
    if k == 2:
        return {"command": "grep -rn \"TODO\" src/ | head -n 20 && echo \"done\\n\"", "timeout": 120000, "description": "find TODOs"}
    return {"query": L._text(rng, 30, escapes=False), "max_results": int(rng.integers(1, 50)), "filters": {"lang": ["py", "go"], "score": 0.25}}


def _tool(rng, k):
    t = {"name": "tool_%d" % k, "description": L._text(rng, int(rng.integers(40, 400))), "input_schema": L._schema(rng)}
    if k % 5 == 1:
        t["type"] = "custom"
    if k % 11 == 7:
        t["input_schema"]["$schema"] = "http://json-schema.org/draft-07/schema#"
    return t


def agent_transcript(seed, target, big_input=0, ntools=None):
    """An Anthropic-format agent request of about `target` bytes; `big_input`: the first tool_use input of an assistant turn holds a
    file body of that size while it fits the target"""
    rng = np.random.default_rng(seed)
    model = MODELS[seed % len(MODELS)]
    sys_text = L._text(rng, max(3000, target // 15))
    system = [{"type": "text", "text": sys_text[: len(sys_text) // 3]}, {"type": "text", "text": sys_text[len(sys_text) // 3:], "cache_control": {"type": "ephemeral"}},
              {"type": "text", "text": "Current date: 2026-10-19"}]
    ntools = ntools or int(rng.integers(10, 41))
    tools = [_tool(rng, k) for k in range(ntools)]
    tools[-1]["cache_control"] = {"type": "ephemeral"}
    msgs = [{"role": "user", "content": [{"type": "text", "text": L._text(rng, 500)}, {"type": "text", "text": "Begin.", "cache_control": {"type": "ephemeral"}}]}]
    size = len(sys_text) + sum(len(json.dumps(t)) for t in tools) + 1000
    ids = 0
    while size < target or ids < 6:
        calls = []
        blocks = [{"type": "text", "text": L._text(rng, int(rng.integers(50, 800)))}] if rng.random() < 0.8 else []
        for _ in range(int(rng.integers(1, 4))):
            ids += 1
            inp = _input(rng, big_input if big_input and not calls and len(msgs) > 1 and size + big_input <= target else 0)
            calls.append(("toolu_%04d" % ids, len(json.dumps(inp))))
            b = {"type": "tool_use", "id": "toolu_%04d" % ids, "name": "tool_%d" % int(rng.integers(ntools)), "input": inp}
            if rng.random() < 0.05:
                b["input"] = None
            blocks.append(b)
            size += calls[-1][1] + 100
        msgs.append({"role": "assistant", "content": blocks if rng.random() < 0.9 else L._text(rng, 300)})
        results = []
        for cid, _ in calls:
            r = {"type": "tool_result", "tool_use_id": cid}
            k = rng.random()
            if k < 0.45:
                r["content"] = _file(rng, int(rng.integers(100, 6000)))
            elif k < 0.8:
                r["content"] = [{"type": "text", "text": L._text(rng, int(rng.integers(50, 3000)))} for _ in range(int(rng.integers(1, 3)))]
            elif k < 0.9:
                r["content"] = None
            else:
                r["content"] = ""
            if rng.random() < 0.3:
                r["is_error"] = bool(rng.random() < 0.5)
            if rng.random() < 0.1:
                r["cache_control"] = {"type": "ephemeral"}
            results.append(r)
            size += len(json.dumps(r.get("content"))) + 80
        if rng.random() < 0.3:
            results.append({"type": "text", "text": L._text(rng, 200)})
        msgs.append({"role": "user", "content": results})
    msgs.append({"role": "assistant", "content": "Done. " + L._text(rng, 100)})
    msgs.append({"role": "user", "content": "Thanks, now summarise."})
    body = {"model": model, "max_tokens": [8192, 4096.0, 1024, 64000.0][seed % 4], "system": system if seed % 3 else sys_text, "messages": msgs, "tools": tools}
    tc = TOOL_CHOICES[seed % len(TOOL_CHOICES)]
    if tc is not None:
        body["tool_choice"] = tc
    if seed % 2:
        body["stream"] = True
    if seed % 3 == 1:
        body["stop_sequences"] = ["\n\nHuman:", "END_TURN"]
    if seed % 4 == 2:
        body["top_k"] = 40
        body["temperature"] = 0.7
    if seed % 5 == 3:
        body["top_p"] = 0.95
        body["metadata"] = {"user_id": "agent-%d" % seed}
    if seed % 4 == 1:
        return json.dumps(body, ensure_ascii=True).encode()
    if seed % 4 == 3:
        return json.dumps(body, indent=1, ensure_ascii=False).encode()
    return json.dumps(body, ensure_ascii=False).encode()


def agent_corpus():
    return [agent_transcript(300 + i, t) for i, t in enumerate(SIZES)]


def big_input_corpus():
    """a single tool_use input of a 1 MiB file body, and a transcript whose inputs total several MiB"""
    one = agent_transcript(401, 1_200_000, big_input=1 << 20)
    several = agent_transcript(402, 5_000_000, big_input=1 << 20)
    return [one, several]


def small_corpus():
    """the generator's requests cut below 64 KiB, for the comparison with the translate pass"""
    return [agent_transcript(604 + i, t, ntools=2 + i) for i, t in enumerate((15_000, 25_000, 35_000, 42_000))]


def inputs_total(body):
    j = json.loads(body)
    return sum(len(json.dumps(b.get("input"), separators=(",", ":"))) for m in j["messages"] if isinstance(m["content"], list)
               for b in m["content"] if b["type"] == "tool_use")


def dense_shapes(n):
    """the densest records per body byte: a user text of \\b escapes (re-spelled as six-byte u-escapes: 3x), runs of the shortest
    tool_result blocks, and tool_use blocks with empty inputs"""
    b1 = b'{"model":"m","messages":[{"role":"user","content":"' + b"\\b" * n + b'"}]}'
    b2 = json.dumps({"model": "m", "messages": [{"role": "user", "content": [{"type": "tool_result", "tool_use_id": "a"}] * max(1, n // 41)}]},
                    separators=(",", ":")).encode()
    b3 = json.dumps({"model": "m", "messages": [{"role": "assistant", "content": [{"type": "tool_use", "id": "a", "name": "n", "input": {}}] * max(1, n // 51)}]},
                    separators=(",", ":")).encode()
    return [b1, b2, b3]


def test_corpus_shape_and_reproducible():
    # pinned: a change to the generators changes what the GPU tests compare, and shows here
    assert L.digest(agent_corpus()) == DIGESTS["agent"]
    assert L.digest(big_input_corpus()) == DIGESTS["big"]
    assert L.digest(small_corpus()) == DIGESTS["small"]
    assert L.digest(dense_shapes(4000)) == DIGESTS["shapes"]
    forms = set()
    for b, t in zip(agent_corpus(), SIZES):
        assert 0.9 * t < len(b) < 1.4 * t, (len(b), t)
        j = json.loads(b)
        assert 10 <= len(j["tools"]) <= 40 and any("properties" in t["input_schema"] for t in j["tools"])
        blocks = [x for m in j["messages"] if isinstance(m["content"], list) for x in m["content"]]
        uses = [x for x in blocks if x["type"] == "tool_use"]
        results = [x for x in blocks if x["type"] == "tool_result"]
        if t >= 150_000:   # the smallest is mostly system prompt and tools
            assert len(uses) >= 3 and any(isinstance(x.get("input"), dict) and any(isinstance(v, dict) for v in x["input"].values()) for x in uses)
            assert {type(x.get("content")).__name__ for x in results} >= {"str", "list"}
        forms.add((b"\\u" in b, b"\n " in b))
    assert forms >= {(True, False), (False, True), (False, False)}
    both = agent_corpus() + small_corpus()
    tcs = {json.dumps(json.loads(b).get("tool_choice"), sort_keys=True) for b in both}
    assert len(tcs) == len(TOOL_CHOICES)
    assert any(isinstance(json.loads(b)["max_tokens"], float) for b in both)
    assert any("top_k" in json.loads(b) for b in both) and any("stop_sequences" in json.loads(b) for b in both)
    assert any(isinstance(json.loads(b)["system"], list) and any("cache_control" in s for s in json.loads(b)["system"]) for b in both)
    assert {json.loads(b)["model"] for b in both} == set(MODELS)
    assert any(b'"content": null' in b or b'"content":null' in b for b in both)
    one, several = big_input_corpus()
    assert max(len(x) for x in (one, several)) < 16 << 20
    assert inputs_total(one) > 1 << 20 and inputs_total(several) > 3 << 20
    assert all(len(b) < 64 << 10 for b in small_corpus())


@pytest.mark.parametrize("schema", SCHEMAS)
@pytest.mark.parametrize("override", ["", OVERRIDE])
def test_oracle_accepts(schema, override):
    bodies = agent_corpus()[:4] + small_corpus() + big_input_corpus()[:1]
    for b in bodies:
        t = oracle(schema, b, override)
        assert t.status == O.OK, (len(b), t.err)
        j = json.loads(t.body)
        m = override or json.loads(b)["model"]
        if schema == "openai":
            assert t.path == "/v1/chat/completions" and j["model"] == m
            assert list(j)[:3] == ["messages", "model", "max_completion_tokens"]
        else:
            assert t.path.startswith("/model/") and t.path.endswith("/converse-stream" if json.loads(b).get("stream") else "/converse")
            assert "messages" in j and "inferenceConfig" in j
        assert t.stream == bool(json.loads(b).get("stream"))


def test_oracle_big_input_is_one_arguments_string():
    one = big_input_corpus()[0]
    t = oracle("openai", one)
    calls = [c for m in json.loads(t.body)["messages"] for c in (m.get("tool_calls") or [])]
    assert max(len(c["function"]["arguments"]) for c in calls) > 1 << 20
    big = max(calls, key=lambda c: len(c["function"]["arguments"]))
    assert json.loads(big["function"]["arguments"])["content"].count("\n") > 1000


def test_oracle_verdicts():
    """the errors the GPU tests place deep in large bodies: a 400 type error after the messages, the Bedrock role 422 after a long
    history, the missing model"""
    base = agent_corpus()[2]
    j = json.loads(base)
    j["temperature"] = "hot"   # a member after the messages
    assert all(oracle(s, json.dumps(j).encode()).status == O.MALFORMED_400 for s in SCHEMAS)
    k = json.loads(base)
    k["messages"].insert(len(k["messages"]) - 1, {"role": "system", "content": "x"})
    assert oracle("aws-bedrock", json.dumps(k).encode()).status == O.INVALID_422
    assert oracle("openai", json.dumps(k).encode()).status == O.OK
    m = json.loads(base)
    del m["model"]
    assert all(oracle(s, json.dumps(m).encode()).status == O.INVALID_422 for s in SCHEMAS)


def test_oracle_record_ratios():
    """the densest shapes give the header's ratio; the host arena (3 * len per body) holds them"""
    b1, b2, b3 = dense_shapes(30000)
    for schema in SCHEMAS:
        r = [len(oracle(schema, b).body) / len(b) for b in (b1, b2, b3)]
        assert 2.95 < r[0] < 3.01 and max(r[1:]) < 1.6, (schema, r)
        for b in (b1, b2, b3):
            t = oracle(schema, b)
            assert len(t.path) + len(t.body) <= 3 * len(b) + 1024
    for b in agent_corpus()[:3] + big_input_corpus()[:1]:
        for schema in SCHEMAS:
            assert len(oracle(schema, b).body) < 1.2 * len(b)


DIGESTS = {"agent": "e6de43c09eac70247a678236ff13c7d55f133b1142580f07b151df9cf5f26c92",
           "big": "0afcba25dfb1610cc2e0f63463f4f37b1a79caa7e27109917f3d97f9afeb5a17",
           "small": "39bd940eec321e50f37fff8cd4d32d15d6b7c6c288225d4ddab2f91c522e0b3e",
           "shapes": "437da39b07e6beb28d0762371e834124089d0749c2beba6a7fa5bbaba0f5abed"}
