"""Corpora of /v1/chat/completions requests for aigw_chat_translate_large_* (test_chat_large_gpu.py feeds them through the GPU):
seeded multi-turn agent transcripts of 64 KiB to 8 MiB, bodies with a feature placed at every thread, warp and tile boundary of
the scan, and bodies at the limits.  Here: their shape, that they are reproducible, and the oracle's verdicts."""
import hashlib
import json

import numpy as np
import pytest

import _oracle as O

TILE, WARP, THREAD = 8192, 1024, 32
WORDS = ("the request handler reads the file and returns its contents to the agent loop which then decides what to call next "
         "while keeping the conversation history in memory so that every turn resends tool results and prior reasoning").split()
STREAM_MODES = ["none", "false", "true", "true_so_null", "true_so_empty", "true_so_other", "true_iu_false", "true_iu_true", "true_iu_null"]


def _text(rng, n, escapes=True):
    out, size = [], 0
    while size < n:
        w = WORDS[int(rng.integers(len(WORDS)))]
        out.append(w); size += len(w) + 1
    s = " ".join(out)[:n]
    if escapes and rng.random() < 0.3:
        s += "\nline two\twith a tab and a \"quote\" and a backslash \\ and café"
    return s


def _schema(rng, depth=0):
    """nested JSON-schema parameters; their strings hold no \\u escape, which the translate pass declines inside parameters"""
    props = {}
    for k in range(int(rng.integers(2, 6))):
        kind = int(rng.integers(4))
        if kind == 0 or depth >= 3:
            props["field_%d" % k] = {"type": "string", "description": _text(rng, 40, escapes=False)}
        elif kind == 1:
            props["count_%d" % k] = {"type": "integer", "minimum": 0, "maximum": 1000}
        elif kind == 2:
            props["items_%d" % k] = {"type": "array", "items": _schema(rng, depth + 1)}
        else:
            props["obj_%d" % k] = _schema(rng, depth + 1)
    return {"type": "object", "properties": props, "required": sorted(props)[:1]}


def _stream_members(mode):
    if mode == "none":
        return {}
    if mode == "false":
        return {"stream": False}
    m = {"stream": True}
    extra = {"true_so_null": None, "true_so_empty": {}, "true_so_other": {"x": 1}, "true_iu_false": {"include_usage": False},
             "true_iu_true": {"include_usage": True}, "true_iu_null": {"include_usage": None}}
    if mode in extra:
        m["stream_options"] = extra[mode]
    return m


def long_chat(seed, target, stream_mode="true", model=True, escaped_args=True):
    """A multi-turn agent transcript of about `target` bytes: a system prompt, user text parts with cache_control, assistant tool
    calls whose JSON arguments are escaped inside their strings, long tool results, and tools with nested JSON-schema parameters."""
    rng = np.random.default_rng(seed)
    tools = [{"type": "function", "function": {"name": "tool_%d" % k, "description": _text(rng, 80), "parameters": _schema(rng)}} for k in range(int(rng.integers(2, 6)))]
    msgs = [{"role": "system", "content": _text(rng, int(rng.integers(500, 4000)))}]
    size, turn = 2000, 0
    while size < target:
        turn += 1
        if rng.random() < 0.5:
            msgs.append({"role": "user", "content": [{"type": "text", "text": _text(rng, int(rng.integers(50, 2000)))},
                                                     {"type": "text", "text": _text(rng, 200), "cache_control": {"type": "ephemeral"}}]})
        else:
            msgs.append({"role": "user", "content": _text(rng, int(rng.integers(50, 2000)))})
        calls = []
        for c in range(int(rng.integers(1, 4))):
            # the arguments text is ASCII, as the translate pass requires of it: its own escapes are \" \\ \n, which the
            # enclosing string escapes once more
            query = " ".join(WORDS[int(x)] for x in rng.integers(0, len(WORDS), 8)) + (' "quoted" \\ and\nmore' if escaped_args else "")
            args = {"path": "/src/module_%d.py" % c, "line": int(rng.integers(1, 999)), "query": query,
                    "options": {"recursive": bool(rng.random() < 0.5), "limit": 50}}
            calls.append({"id": "call_%d_%d" % (turn, c), "type": "function", "function": {"name": "tool_%d" % int(rng.integers(len(tools))), "arguments": json.dumps(args)}})
        msgs.append({"role": "assistant", "content": None if rng.random() < 0.5 else _text(rng, 120), "tool_calls": calls})
        for c in calls:
            res = _text(rng, int(rng.integers(2000, max(4000, target // 40))))
            msgs.append({"role": "tool", "tool_call_id": c["id"], "content": res})
            size += len(res) + 200
        size += 3000
    body = {}
    if model:
        body["model"] = "gpt-4o-mini"
    body["messages"] = msgs
    body["tools"] = tools
    body["tool_choice"] = "auto"
    body["temperature"] = 0.2
    body["max_completion_tokens"] = 4096
    body.update(_stream_members(stream_mode))
    return json.dumps(body, separators=(",", ":") if seed % 2 else (", ", ": ")).encode()


def realistic_corpus(n=18, lo=64 << 10, hi=8 << 20):
    """sizes spread log-uniformly between 64 KiB and 8 MiB, every stream mode, some without a model"""
    rng = np.random.default_rng(1234)
    out = []
    for i in range(n):
        target = int(np.exp(rng.uniform(np.log(lo), np.log(hi))))
        out.append(long_chat(100 + i, target, STREAM_MODES[i % len(STREAM_MODES)], model=i % 5 != 4))
    return out


def boundary_bodies():
    """One feature (an escape, a key, a number, a quote) placed within +-40 bytes of each thread, warp and tile boundary of the scan."""
    out = []
    base = long_chat(7, 20000, "true")
    for edge in (THREAD, WARP, TILE, 2 * TILE, 3 * TILE):
        for delta in range(-40, 41, 3):
            pad = edge + delta - len(b'{"model":"m","x":"') - 1
            if pad < 0:
                continue
            for feat in (b'\\"', b'\\\\', b'\\u00e9', b'\\/'):
                s = b'{"model":"m","x":"' + b"a" * pad + feat + b'","messages":[{"role":"user","content":"hi"}],"stream":true}'
                out.append(s)
            # a key straddling the edge, followed by the real body
            out.append(b'{"' + b"k" * max(1, edge + delta - 2) + b'":1,' + base[1:])
    return out


def limit_bodies():
    """nesting depth 48 and 49 under a member the request ignores"""
    def deep(d):
        v = "1"
        for _ in range(d - 1):
            v = '{"a":' + v + "}"
        return ('{"model":"m","messages":[{"role":"user","content":"hi"}],"x":' + v + "}").encode()
    return deep(48), deep(49)


def near_16mib():
    body = long_chat(9, 256 << 10, "true")
    k = (16 << 20) - 1 - len(body) - 10
    return body[:-1] + b',"user":"' + b"u" * k + b'"}'


def digest(bodies):
    h = hashlib.sha256()
    for b in bodies:
        h.update(len(b).to_bytes(8, "little")); h.update(b)
    return h.hexdigest()


def test_corpus_shape_and_reproducible():
    c = realistic_corpus()
    # pinned: a change to the generator changes what the GPU tests compare, and shows here
    assert digest(c) == "2e7b5750c259341e92d59a6fb32bb531316340c59491bd075e947e61d6b96fb0"
    assert digest(boundary_bodies()) == "5172c8a83eb196b0a2c426015ef5cee585f0faef8c5af623cd096b4d88f9d132"
    sizes = [len(b) for b in c]
    assert min(sizes) >= 64 << 10 and max(sizes) <= 9 << 20 and max(sizes) >= 2 << 20, sizes
    for b in c:
        j = json.loads(b)
        roles = {m["role"] for m in j["messages"]}
        assert roles == {"system", "user", "assistant", "tool"}
        assert any("cache_control" in p for m in j["messages"] if isinstance(m.get("content"), list) for p in m["content"])
        assert any("\\\"" in m["tool_calls"][0]["function"]["arguments"] or '"' in m["tool_calls"][0]["function"]["arguments"]
                   for m in j["messages"] if m["role"] == "assistant")
    assert b"\\\"" in c[0]   # escaped quotes inside the arguments strings


def test_boundary_and_limit_shapes():
    bb = boundary_bodies()
    assert len(bb) > 100 and all(json.loads(b) is not None for b in bb)
    d48, d49 = limit_bodies()
    assert json.loads(d48) and json.loads(d49)
    big = near_16mib()
    assert len(big) == (16 << 20) - 1 and json.loads(big)["model"] == "gpt-4o-mini"


@pytest.mark.parametrize("schema,override,cost", [("openai", "", True), ("openai", "ovr-model", False), ("azure-openai", "", True), ("azure-openai", "dep", False)])
def test_oracle_accepts_realistic(schema, override, cost):
    for b in realistic_corpus(9, hi=2 << 20):
        t = O.chat_translate(schema, b, model_override=override, cost_configured=cost, prefix="2025-01-01-preview" if schema == "azure-openai" else "v1")
        assert t.status == O.OK, (schema, len(b), t.err)
        if schema == "azure-openai":
            assert t.path.startswith("/openai/deployments/")
        elif override:
            assert t.body_kind == O.BYTES


def test_oracle_verdicts_limits():
    d48, d49 = limit_bodies()
    assert O.chat_translate("openai", d48).status == O.OK
    big = near_16mib()
    assert O.chat_translate("openai", big, cost_configured=True).status == O.OK
