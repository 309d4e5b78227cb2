"""Corpora of /v1/embeddings requests for aigw_embeddings_translate_large_* (test_embeddings_large_gpu.py feeds them through the
GPU), and a small restatement of the three translations (OpenAI passthrough, Vertex predict, Titan) from json.loads and a Go-style
string encoder, checked against the oracle here so that the oracle is not the only judge of the re-encoding."""
import json
import random

import pytest

import _oracle as O

TASKS = ["RETRIEVAL_QUERY", "RETRIEVAL_DOCUMENT", "SEMANTIC_SIMILARITY", "CLUSTERING", ""]
WORDS = ["refund", "policy", "café", "日本語のテキスト", "emoji 😀 here", "line\nbreak", 'quo"te', "tab\there", "back\\slash", "a/b", "\x08bell\x0c",
         "vector", "search", "embedding", "Ωmega", "naïve"]


def _text(r, lo, hi):
    out, n, have = [], r.randint(lo, hi), 0
    while have < n:
        w = r.choice(WORDS) if r.random() < 0.3 else "w%d" % r.randint(0, 99999)
        out.append(w); have += len(w) + 1
    return " ".join(out)[:n] or "x"


def _dump(d, r, variant):
    if variant == "ascii":
        return json.dumps(d, ensure_ascii=True, separators=(",", ":")).encode()
    if variant == "indent":
        return json.dumps(d, ensure_ascii=False, indent=2).encode()
    return json.dumps(d, ensure_ascii=False, separators=(",", ":")).encode()


def large_corpus(seed=11, total=24 << 20):
    """realistic requests of 64 KiB to 8 MiB: string batches, ensure_ascii / indent variants, token ids, items, request-level
    fields, single long strings (the Titan shape)"""
    r = random.Random(seed)
    out, size, k = [], 0, 0
    while size < total:
        shape = k % 6
        k += 1
        variant = ("", "ascii", "indent")[r.randint(0, 2)]
        d = {"model": r.choice(["text-embedding-3-small", "text-embedding-004", "amazon.titan-embed-text-v2:0"])}
        if shape == 0:
            d["input"] = [_text(r, 50, 2000) for _ in range(r.randint(100, 600))]
        elif shape == 1:
            d["input"] = [r.randint(100, 999999) for _ in range(r.randint(20000, 60000))]
        elif shape == 2:
            d["input"] = [[r.randint(100, 999999) for _ in range(r.randint(50, 400))] for _ in range(r.randint(40, 200))]
        elif shape == 3:
            d["input"] = [{k2: v for k2, v in {"content": _text(r, 50, 3000) if r.random() < 0.7 else [_text(r, 20, 800) for _ in range(r.randint(1, 4))],
                                              "task_type": r.choice(TASKS) if r.random() < 0.7 else None,
                                              "title": _text(r, 5, 60) if r.random() < 0.6 else None}.items() if v is not None} for _ in range(r.randint(100, 500))]
        elif shape == 4:
            d["input"] = [_text(r, 50, 8000) if r.random() < 0.95 else None for _ in range(r.randint(100, 400))]
            d["task_type"] = r.choice(TASKS[:4]); d["auto_truncate"] = r.random() < 0.5; d["dimensions"] = r.choice([0, 256, 768, -1])
        else:
            d["input"] = _text(r, 1 << 20, 3 << 20)
            if r.random() < 0.5: d["dimensions"] = 512
        if r.random() < 0.3:
            d = dict(reversed(list(d.items())))   # the model after megabytes of input
        b = _dump(d, r, variant)
        if 65536 < len(b) <= 8 << 20:
            out.append(b); size += len(b)
    return out


def titan_bodies(seed=5):
    """single 1-16 MiB strings (Titan's one input), plain and with ensure_ascii escapes"""
    r = random.Random(seed)
    out = []
    for n, ascii_ in ((1 << 20, False), (3 << 20, True), (6 << 20, True), ((16 << 20) - 4096, False)):
        s = "".join(r.choice(WORDS) + " " for _ in range(n // 12))
        b = json.dumps({"model": "amazon.titan-embed-text-v2:0", "input": s}, ensure_ascii=ascii_).encode()
        while len(b) >= 16 << 20:
            s = s[:len(s) - (len(b) - (16 << 20)) - 64]
            b = json.dumps({"model": "amazon.titan-embed-text-v2:0", "input": s}, ensure_ascii=ascii_).encode()
        out.append(b)
    return out


# a feature placed inside the first input string at a given offset (the offset of the feature's first byte)
FEATURES = {
    "run_bs2_quote": b'\\\\\\\\\\"', "run_bs1": b"\\\\", "esc_slash": b"\\/", "esc_b": b"\\b", "esc_f": b"\\f", "esc_n": b"\\n",
    "u_escape": b"\\u00e9", "u_ctrl": b"\\u001F", "u_quote": b"\\u0022", "surrogate": b"\\ud83d\\ude00", "lone_high": b"\\ud83d x",
    "lone_low": b"x \\ude00", "bad_hex": b"\\u12g4", "bs_u_literal": b"\\\\ud83d\\ude00",
}
OK_FEATURES = ("run_bs2_quote", "run_bs1", "esc_slash", "esc_b", "esc_f", "esc_n", "u_escape", "u_ctrl", "u_quote", "surrogate")


def feature_body(feature, at, length=20000):
    head = b'{"model":"m","input":["'
    f = FEATURES[feature]
    pre = b"a" * max(0, at - len(head))
    first = pre + f
    rest = length - len(head) - len(first) - 4
    tail = b'","' + b"b" * max(1, rest // 2) + b'"]}'
    return head + first + tail


def boundary_corpus(window=40, step=7):
    out = []
    for bound in (32, 1024, 8192, 16384):
        for name in FEATURES:
            for at in range(bound - window, bound + window, step):
                out.append(("%s @%d" % (name, at), feature_body(name, at)))
        for at in range(bound - window, bound + window, step):   # null / number / nested elements, the model member
            pad = b"x" * max(1, at - 24)
            out.append(("null_elem @%d" % at, b'{"model":"m","input":["' + pad + b'",null,"y"]}'))
            out.append(("number_elem @%d" % at, b'{"model":"m","input":["' + pad + b'",5,"y"]}'))
            out.append(("nested_elem @%d" % at, b'{"model":"m","input":["' + pad + b'",["y"]]}'))
            out.append(("model @%d" % at, b'{"input":["' + pad + b'"],"model":"mm"}'))
    return out


def splice_corpus():
    big = json.dumps(["chunk %d " % i + "x" * 500 for i in range(5000)], separators=(",", ":"))
    return [
        ('{"input":%s,"model":"text-embedding-3-small"}' % big).encode(),   # the model last, after megabytes of input
        ('{"input":%s}' % big).encode(),                                    # no model: the member is appended
        ('{"model":null,"input":%s}' % big).encode(),                       # a null model is replaced
        b"{}", b"null", b'{"model":"m","input":"a"}', b' {"input":"a"} ',
    ]


# ---------------------------------------------------------------- the restatement
def go_str(s):
    """encoding/json's spelling of a string, without HTML escaping"""
    out = ['"']
    for ch in s:
        o = ord(ch)
        if ch == '"': out.append('\\"')
        elif ch == "\\": out.append("\\\\")
        elif ch == "\n": out.append("\\n")
        elif ch == "\r": out.append("\\r")
        elif ch == "\t": out.append("\\t")
        elif o < 0x20: out.append("\\u%04x" % o)
        else: out.append(ch)
    out.append('"')
    return "".join(out)


def restate(schema, body, override=""):
    """(path, body bytes or None) of the translation of a request the oracle accepts, for a realistic request (no duplicate keys,
    well-typed); None when the target declines it with a 422 / 500"""
    d = json.loads(body)
    model = override or d.get("model") or ""
    inp = d.get("input")
    if schema == "openai":
        return "/v1/embeddings", None
    if schema == "aws-bedrock":
        if isinstance(inp, str): text = inp
        elif isinstance(inp, list) and len(inp) == 1 and (inp[0] is None or isinstance(inp[0], str)): text = inp[0] or ""
        else: return None
        from urllib.parse import quote
        path = "/model/%s/invoke" % quote(model, safe="-_.~$&+:=@")
        out = '{"inputText":' + go_str(text) + ("" if d.get("dimensions") is None else ',"dimensions":%s' % json.dumps(d["dimensions"])) + "}"
        return path, out.encode()
    gtask = d.get("task_type") or None
    inst = []
    def one(c, task, title):
        s = '{"content":' + go_str(c or "")
        if task: s += ',"task_type":' + go_str(task)
        if title is not None: s += ',"title":' + go_str(title)
        inst.append(s + "}")
    def item(it):
        task, title = it.get("task_type"), it.get("title")
        keep = task == "RETRIEVAL_DOCUMENT" and title
        c = it.get("content")
        for x in (c if isinstance(c, list) else [c]):
            one(x, gtask or task, title if keep else None)
    if isinstance(inp, str): one(inp, gtask, None)
    elif isinstance(inp, dict): item(inp)
    elif isinstance(inp, list) and inp and isinstance(inp[0], dict):
        for it in inp: item(it)
    elif isinstance(inp, list) and all(x is None or isinstance(x, str) for x in inp):
        for x in inp: one(x, gtask, None)
    else:
        return None
    params = []
    if d.get("auto_truncate") is True: params.append('"auto_truncate":true')
    if isinstance(d.get("dimensions"), int) and d["dimensions"] > 0: params.append('"outputDimensionality":%d' % d["dimensions"])
    out = '{"instances":' + ("[" + ",".join(inst) + "]" if inst else "null") + ',"parameters":{' + ",".join(params) + "}}"
    return "publishers/google/models/%s:predict" % model, out.encode()


def test_generators_are_deterministic():
    assert large_corpus(total=4 << 20) == large_corpus(total=4 << 20)
    assert boundary_corpus() == boundary_corpus()
    assert [len(b) for b in titan_bodies()] == [len(b) for b in titan_bodies()]


def test_corpus_shapes():
    bodies = large_corpus()
    assert all(65536 < len(b) <= 8 << 20 for b in bodies) and sum(map(len, bodies)) >= 24 << 20
    assert all(len(b) < 16 << 20 for b in titan_bodies())
    assert all(len(b) > 20 for _, b in boundary_corpus())


@pytest.mark.parametrize("schema", ["gcp-vertexai", "aws-bedrock", "openai"])
def test_restatement_agrees_with_oracle(schema):
    bodies = large_corpus(total=8 << 20) + [b for b in titan_bodies()[:2]]
    bodies += [b for l, b in boundary_corpus() if l.split()[0] in OK_FEATURES][::5]
    n = 0
    for b in bodies:
        for override in ("", "text-embedding-005"):
            t = O.embeddings_translate(schema, b, model_override=override)
            want = restate(schema, b, override)
            if want is None:
                assert t.status != O.OK, b[:200]
                continue
            assert t.status == O.OK, (b[:200], t.err)
            path, out = want
            assert t.path == path, (t.path, path)
            if out is not None:
                assert t.body == out, (b[:200], t.body[:300], out[:300])
            n += 1
    assert n >= 4
