"""The /v1/responses request oracle (tests/_responses_request_oracle.py) against the reference's own answers, and the corpus
generators the GPU test (test_responses_request_gpu.py) feeds through every entry point.

Goldens: tests/golden/responses_request_cases.json (lifted by extract_responses_request_goldens.py) and the data-plane requests
"openai - /v1/responses" / "- stream" of testupstream_cases.json."""
import base64
import json
import os
import random

import _responses_request_oracle as Q
import test_translate_edges_cpu as E

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "responses_request_cases.json"), encoding="utf-8"))
UPSTREAM = {c["name"]: c for c in json.load(open(os.path.join(HERE, "golden", "testupstream_cases.json"), encoding="utf-8"))["cases"]}
MAX_BODY = 65536   # the translate pass's largest size class


# ================================================================ realistic corpus: multi-turn agent requests
WORDS = ("the tool returned an error so I will retry with a smaller page size; results are listed below, grouped by file "
         "naïve café – 日本語のテキスト — ünïcödé \"quoted\" path\\to\\file\nnew line\ttab").split(" ")
TOOL_NAMES = ("read_file", "write_file", "run_shell", "search_code", "list_dir", "apply_patch_text", "web_fetch", "get_weather")


def _text(r, lo, hi):
    n = int(r.lognormvariate(0, 1.0) * (lo + hi) / 4)
    return " ".join(r.choice(WORDS) for _ in range(max(lo, min(hi, n))))


def _tool(r, name):
    props = {f"arg{k}": {"type": r.choice(("string", "integer", "boolean")), "description": _text(r, 8, 40)} for k in range(r.randint(1, 4))}
    t = {"type": "function", "name": name, "description": _text(r, 30, 120),
         "parameters": {"type": "object", "properties": props, "required": sorted(props)[:r.randint(0, len(props))], "additionalProperties": False}}
    if r.random() < 0.5:
        t["strict"] = True
    return t


def _item(r, k, turn):
    kind = r.choices(("easy", "typed_user", "assistant", "call", "reasoning"), (3, 2, 3, 4, 2))[0]
    if kind == "easy":
        return [{"role": r.choice(("user", "developer", "system")), "content": _text(r, 3, 200)}]
    if kind == "typed_user":
        parts = [{"type": "input_text", "text": _text(r, 3, 120)}]
        if r.random() < 0.15:
            parts.append({"type": "input_image", "image_url": "https://example.com/img/%d.png" % turn, "detail": "auto"})
        if r.random() < 0.05:
            parts.append({"type": "input_file", "file_id": "file-%06d" % turn, "filename": "notes.txt"})
        return [{"type": "message", "role": "user", "content": parts}]
    if kind == "assistant":
        m = {"type": "message", "role": "assistant", "content": [{"type": "output_text", "text": _text(r, 3, 300), "annotations": []}]}
        if r.random() < 0.7:
            m["id"] = "msg_%016x" % r.getrandbits(64)
            m["status"] = "completed"
        return [m]
    if kind == "reasoning":
        blob = base64.b64encode(r.randbytes(r.choice((256, 1024, 3072, 6144)))).decode()
        return [{"type": "reasoning", "id": "rs_%016x" % r.getrandbits(64), "summary": [{"type": "summary_text", "text": _text(r, 3, 80)}] if r.random() < 0.6 else [],
                 "encrypted_content": blob}]
    call_id = "call_%012x" % r.getrandbits(48)
    args = json.dumps({"path": "src/%s.py" % r.choice(WORDS).strip('"\\\n\t'), "limit": r.randint(1, 500)})
    fc = {"type": "function_call", "call_id": call_id, "name": r.choice(TOOL_NAMES), "arguments": args}
    if r.random() < 0.6:
        fc["id"] = "fc_%016x" % r.getrandbits(64)
        fc["status"] = "completed"
    return [fc, {"type": "function_call_output", "call_id": call_id, "output": _text(r, 1, 600)}]


def realistic_request(seed, cap=True):
    """One agent-loop turn: instructions, tools, include, store / stream, reasoning, text, and 1-40 input items.  With `cap`, the
    oldest items are dropped until the body fits the 64 KiB size class (a client would start a new conversation instead)."""
    r = random.Random(seed)
    items = []
    for k in range(r.randint(1, 40)):
        items += _item(r, k, seed)
    req = {"model": r.choice(("gpt-5", "gpt-5-codex", "o4-mini", "gpt-4.1")), "instructions": _text(r, 10, 400)}
    if r.random() < 0.8:
        req["tools"] = [_tool(r, n) for n in r.sample(TOOL_NAMES, r.randint(1, 6))]
        req["tool_choice"] = r.choice(("auto", "required", "none", {"type": "function", "name": req["tools"][0]["name"]}))
        req["parallel_tool_calls"] = r.random() < 0.5
    if r.random() < 0.7:
        req["include"] = ["reasoning.encrypted_content"]
    req["store"] = False
    req["stream"] = r.random() < 0.7
    if r.random() < 0.7:
        req["reasoning"] = {"effort": r.choice(("minimal", "low", "medium", "high")), "summary": "auto"}
    if r.random() < 0.5:
        req["text"] = {"verbosity": r.choice(("low", "medium", "high"))}
        if r.random() < 0.3:
            req["text"]["format"] = {"type": "json_schema", "name": "answer", "schema": {"type": "object", "properties": {"a": {"type": "string"}}}, "strict": True}
    if r.random() < 0.3:
        req["max_output_tokens"] = r.randint(256, 32768)
    if r.random() < 0.3:
        req["prompt_cache_key"] = "session-%08x" % r.getrandbits(32)
    if r.random() < 0.2:
        req["metadata"] = {"trace": "t%d" % seed}
    ascii_only = r.random() < 0.3
    while True:
        req["input"] = items
        body = json.dumps(req, ensure_ascii=ascii_only, separators=None if r.random() < 0.3 else (",", ":")).encode()
        if not cap or len(body) <= MAX_BODY or len(items) <= 1:
            return body
        items = items[1:]


def realistic_corpus(n=2000, seed=7):
    return [realistic_request(seed * 100003 + i) for i in range(n)]


def uncapped_share_above(n=2000, seed=7):
    return sum(len(realistic_request(seed * 100003 + i, cap=False)) > MAX_BODY for i in range(n)) / n


# ================================================================ edge corpus
BASE = {"model": "m", "input": [{"role": "user", "content": "hi"}]}
MEMBERS = {   # restated top-level member → a valid value
    "background": True, "parallel_tool_calls": False, "store": False, "stream": True, "max_output_tokens": 100, "max_tool_calls": 3, "top_logprobs": 2,
    "temperature": 0.5, "top_p": 1, "presence_penalty": 0.25, "frequency_penalty": -1, "instructions": "be brief", "previous_response_id": "resp_1",
    "prompt_cache_key": "k", "safety_identifier": "s", "user": "u", "prompt_cache_retention": "24h", "service_tier": "auto", "truncation": "auto",
    "model": "gpt-5", "include": ["reasoning.encrypted_content"], "metadata": {"a": "b"}, "conversation": {"id": "conv_1"},
    "stream_options": {"include_obfuscation": False}, "reasoning": {"effort": "low", "generate_summary": "auto", "summary": "concise"},
    "text": {"verbosity": "low", "format": {"type": "json_object"}}, "tool_choice": {"type": "function", "name": "f"},
    "tools": [{"type": "function", "name": "f", "parameters": {"type": "object"}, "strict": True, "description": "d"}],
    "input": [{"type": "function_call", "call_id": "c", "name": "f", "arguments": "{}"}, {"type": "function_call_output", "call_id": "c", "output": "ok"}],
}
WRONG = [1, 1.5, "s", True, [], {}, [1], {"a": 1}, -0.0]
ITEMS = [
    {"role": "user", "content": "x"}, {"role": "user", "content": [{"type": "input_text", "text": "t"}]},
    {"type": "message", "role": "developer", "content": [{"type": "input_text", "text": "t"}], "status": "completed", "id": "m1"},
    {"type": "message", "role": "assistant", "content": [{"type": "output_text", "text": "a", "annotations": []}, {"type": "refusal", "refusal": "no"}]},
    {"type": "message", "role": "assistant", "content": "plain"},
    {"type": "function_call", "call_id": "c", "name": "f", "arguments": "{}", "id": "fc", "status": "completed"},
    {"type": "function_call_output", "call_id": "c", "output": "o"},
    {"type": "reasoning", "id": "r", "summary": [{"type": "summary_text", "text": "s"}], "encrypted_content": "QUJD", "content": [{"type": "reasoning_text", "text": "x"}]},
    {"type": "item_reference", "id": "ref"},
    {"role": "user", "content": [{"type": "input_image", "image_url": "u", "detail": "low"}, {"type": "input_file", "file_data": "ZA==", "filename": "f"}]},
]


def _dump(o):
    return json.dumps(o, separators=(",", ":")).encode()


def edge_corpus():
    out = []
    for k, v in MEMBERS.items():
        out.append(_dump(dict(BASE, **{k: v})))
        out.append(_dump(dict(BASE, **{k: None})))
        out.append(_dump(dict(BASE, **{k: v, "unknown_" + k: {"x": [1]}})))
        for w in WRONG:
            out.append(_dump(dict(BASE, **{k: w})))
        b = _dump(dict(BASE, **{k: v}))   # the member twice
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(v)))
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(WRONG[0])))
    for it in ITEMS:
        out.append(_dump(dict(BASE, input=[it])))
        out.append(_dump(dict(BASE, input=[dict(it, extra={"deep": [None]})])))
        for key in it:
            for w in [None] + WRONG[:6]:
                out.append(_dump(dict(BASE, input=[dict(it, **{key: w})])))
        s = _dump(it)
        out.append(_dump(BASE)[:-2] + b"," + s[:-1] + b',"type":"message"}]}')   # a second tag
        out.append(b'{"model":"m","input":[{"ty\\u0070e":"message","role":"user","content":"x"}]}')
    for tag in ("file_search_call", "computer_call", "web_search_call", "custom_tool_call", "mcp_call", "compaction", "no_such_item", "", "\\u006dessage"):
        out.append(b'{"model":"m","input":[{"type":"%s","role":"user","content":"x"}]}' % tag.encode())
    for tag in ("web_search", "file_search", "mcp", "custom", "no_such_tool"):
        out.append(b'{"model":"m","tools":[{"type":"%s","name":"n"}]}' % tag.encode())
        out.append(b'{"model":"m","tool_choice":{"type":"%s"}}' % tag.encode())
    out += [b'{"model":"m","instructions":["a"]}', b'{"model":"m","instructions":[]}', b'{"model":"m","text":{"format":null}}',
            b'{"model":"m","text":{"format":{"type":"json_schema","name":"n","schema":{"a\\u0062":[1]}}}}', b'{"model":"m","tools":[null]}',
            b'{"model":"m","input":[null]}', b'{"model":"m","input":[1]}', b'{"model":"m","input":{}}', b'{"model":"m","input":null}',
            b'{"model":"m","input":[{"type":null,"role":"user","content":null}]}', b'{"model":"m","input":[{"type":5,"role":"user","content":"x"}]}',
            b'{"model":"m","input":[{"type":"message","role":"assistant","content":null}]}', b'{"mod\\u0065l":"m"}', b'{"model":"m\\u0065"}',
            b'{"model":"m","prompt":{"id":"p"}}', b'{"model":"m","prompt":null}', b'{"model":"m","context_management":[]}', b'null', b'[]', b'"s"', b'{}',
            b' {"model":"m"} ', b'{"model":"m"} x', b'{"model":"m","max_output_tokens":1234567890123456789}', b'{"model":"m","max_output_tokens":-0}',
            b'{"model":"m","max_output_tokens":1e3}', b'{"model":"m","presence_penalty":1e-3}', b'{"model":"m","temperature":1e-3}',
            b'{"model":"m","metadata":{"k\\u0031":"v"}}', b'{"model":"m","metadata":{"k":1}}', b'{"model":"m","include":[null,"a"]}',
            b'{"model":"m","input":[{"type":"message","role":"assistant","content":[{"type":"output_text","text":"a","annotations":[{"type":"url_citation"}]}]}]}',
            b'{"model":"m","input":[{"type":"function_call_output","call_id":"c","output":[{"type":"input_text","text":"t"}]}]}',
            b'{"model":"m","input":[{"type":"reasoning","id":"r","summary":[null,{"text":"s"}]}]}', b'{"model":"m","input":[{"type":"reasoning","id":"r","summary":[1]}]}',
            b'{"input":"hi"}', b' {"input":[{"role":"user","content":"x"}],"stream":true} \n', b'{"model":null,"input":"hi"}',
            b'{"model":"m","conversation":"conv_1"}', b'{"model":"m","conversation":{"id":5}}', b'{"model":"m","tool_choice":"whatever"}',
            b'{"model":"m","tool_choice":{"name":"f"}}', b'{"model":"m","input":"a\x01b"}', b'{"model":"m","tools":[{"type":"function","parameters":[1]}]}']
    return out


def class_bound_bodies():
    """bodies of exactly c-1, c and c+1 bytes for every size class bound, and one over 64 KiB"""
    out = []
    for c in E.CLASSES:
        for n in (c - 1, c, c + 1):
            head = b'{"model":"m","stream":true,"input":[{"role":"user","content":"'
            tail = b'"}]}'
            out.append(head + b"a" * (n - len(head) - len(tail)) + tail)
    return out


MUTATION_SEEDS = 30


def mutation_seeds():
    r = random.Random(11)
    small = [b for b in realistic_corpus(400, seed=3) if len(b) < 1500]
    return [_dump(dict(BASE, input=[it])) for it in ITEMS] + r.sample(small, min(len(small), MUTATION_SEEDS - len(ITEMS)))


# ================================================================ tests
def test_union_goldens():
    """each UnmarshalJSON case, placed in the request member that decodes it: what the reference decodes is OK or outside the
    subset, what it rejects is a failure or outside the subset"""
    seen = set()
    for u in GOLD["unions"]:
        v, _, _ = Q.parse_body(u["wrapped"].encode())
        assert v != (Q.OK if u["error"] else Q.FAIL), (u["test"], u["name"], v)
        seen.add((u["test"], v))
    assert len(GOLD["unions"]) >= 70
    assert any(v == Q.OK for _, v in seen) and any(v == Q.FAIL for _, v in seen)


def test_parse_body_goldens():
    for c in GOLD["parse_body"]:
        v, model, stream = Q.parse_body(c["body"].encode())
        if c["error"]:
            assert v == Q.FAIL, c["name"]
        else:
            assert (v, model.decode(), stream) == (Q.OK, c["model"], c["stream"]), c["name"]


def test_request_body_goldens():
    for c in GOLD["request_body"]:
        v, path, out, model, stream = Q.translate(c["body"].encode(), c["override"], "v1", c["force"])
        assert v == Q.OK and path == c["exp_path"] and stream == c.get("stream", False), c["name"]
        if "exp_model_member" in c:
            assert json.loads(out)["model"] == c["exp_model_member"], c["name"]
        else:
            assert out == (None if c["exp_body"] is None else c["body"].encode()), c["name"]


def test_data_plane_requests():
    for name in ("openai - /v1/responses", "openai - /v1/responses - stream"):
        c = UPSTREAM[name]
        v, path, out, model, stream = Q.translate(c["requestBody"].encode())
        assert (v, path, out, model, stream) == (Q.OK, c["expPath"], None, b"something", name.endswith("stream")), name


def test_oracle_known_answers():
    cases = {
        b'{"model":"m","input":[{"role":"user","content":"x"}]}': Q.OK,
        b'{"model":"m","input":[{"type":"message","role":"assistant","content":[{"type":"input_text","text":"x"}]}]}': Q.OUT,
        b'{"model":"m","input":[{"type":"message","role":"user","content":[{"type":"output_text","text":"x"}]}]}': Q.OUT,
        b'{"model":"m","instructions":["a"]}': Q.FAIL,
        b'{"model":"m","max_output_tokens":"5"}': Q.FAIL,
        b'{"model":"m","max_output_tokens":1.5}': Q.FAIL,
        b'{"model":"m","max_output_tokens":-0}': Q.OUT,
        b'{"model":"m","input":[{"content":"x"}]}': Q.OUT,
        b'{"model":"m","input":[{"type":"","role":"user","content":"x"}]}': Q.OK,
        b'{"model":"m","input":[{"role":"user","content":"x","role":5}]}': Q.OUT,
        b'{"model":"m","input":[{"role":5,"content":"x"}]}': Q.FAIL,
        b'{"model":"m","input":[{"type":"item_reference","id":"a","zz":{"q":[1,{}]}}]}': Q.OK,
        b'{"model":"m","tools":[{"type":"web_search"}],"max_output_tokens":"x"}': Q.OUT,
        b'{"model":"m","max_output_tokens":"x","tools":[{"type":"web_search"}]}': Q.FAIL,
        b'{"model":"m","tool_choice":null,"conversation":null,"input":null,"text":{"format":{"type":"text"}}}': Q.OK,
        b'{"model":"m","tools":[{"type":"function","parameters":{"a\\u0062":1}}]}': Q.OK,
        b'null': Q.OUT, b'[]': Q.FAIL, b'{"model":"m"}x': Q.FAIL,
    }
    for body, exp in cases.items():
        assert Q.parse_body(body)[0] == exp, body
    assert Q.request_path("") == "/responses" and Q.request_path("/custom/api/") == "/custom/api/responses"
    v, path, out, _, _ = Q.translate(b' {"input":"x"} ', "o-1")
    assert (v, out) == (Q.OK, b'{"input":"x","model":"o-1"}')   # sjson appends at the root and drops the bytes outside it


def test_realistic_corpus_generator():
    bodies = realistic_corpus(400)
    assert len(set(bodies)) == len(bodies)
    assert all(len(b) <= MAX_BODY for b in bodies)
    assert all(Q.parse_body(b)[0] == Q.OK for b in bodies)
    assert {E.class_of(len(b)) for b in bodies} == set(E.CLASSES)   # every size class is represented
    for b in bodies:   # the index stage's token capacity of the body's own class and of the fused kernel
        t = E.count_tokens(b)
        assert t <= E.KTOK[E.class_of(len(b))] and (len(b) > E.SMALL_MAX or t <= E.SMALL_KTOK), (len(b), t)
    kinds = b"".join(bodies)
    for needle in (b'"type":"reasoning"', b'"encrypted_content"', b'"function_call_output"', b'"role":"assistant"', b'"input_text"',
                   b'"include":["reasoning.encrypted_content"]', b'"store":false', b'"stream":true', b'"verbosity"'):
        assert needle in kinds or needle.replace(b":", b": ") in kinds, needle


def test_edge_corpus_generator():
    bodies = edge_corpus()
    verdicts = [Q.parse_body(b)[0] for b in bodies]
    assert {Q.OK, Q.FAIL, Q.OUT} <= set(verdicts)
    assert Q.parse_body(b'{"model":"m","input":[{"role":"user","content":"hi"}],"store":false,"unknown_store":{"x":[1]}}')[0] == Q.OK
    for b in class_bound_bodies():
        assert Q.parse_body(b)[0] == Q.OK
    assert sorted({len(b) for b in class_bound_bodies()})[-1] == MAX_BODY + 1
