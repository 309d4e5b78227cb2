"""Corpora of /v1/responses requests for aigw_responses_translate_large_* (test_responses_large_gpu.py feeds them through the GPU):
seeded agent sessions of 64 KiB to 8 MiB, bodies with a feature placed at every thread, warp and tile boundary of the scan, bodies
at the limits, and probes with malformed bytes on those boundaries.  Here: their shape, that they are reproducible, and the
oracle's verdicts."""
import functools
import hashlib
import json
import random

import _responses_request_oracle as Q
import test_large_scan_defects_cpu as D
import test_responses_request_cpu as G

TILE, WARP, THREAD = 8192, 1024, 32
STREAM_FORMS = ("absent", "false", "true", "null")


def long_session(seed, target, stream="true"):
    """An agent session of about `target` bytes: instructions, function tools, and a transcript of input items from
    test_responses_request_cpu's _item, with more turns, file-sized function_call_output strings and multi-KB encrypted_content."""
    r = random.Random(seed)
    req = {"model": r.choice(("gpt-5", "gpt-5-codex", "o4-mini")), "instructions": G._text(r, 200, 1500)}
    req["tools"] = [G._tool(r, n) for n in r.sample(G.TOOL_NAMES, r.randint(2, 8))]
    req["tool_choice"] = r.choice(("auto", "required", {"type": "function", "name": req["tools"][0]["name"]}))
    req["include"] = ["reasoning.encrypted_content"]
    req["store"] = False
    req["reasoning"] = {"effort": r.choice(("low", "medium", "high")), "summary": "auto"}
    if stream != "absent":
        req["stream"] = {"false": False, "true": True, "null": None}[stream]
    items, size, turn = [], 0, 0
    while size < target:
        turn += 1
        for it in G._item(r, turn, seed):
            if it.get("type") == "function_call_output" and r.random() < 0.5:   # a file read back to the model
                it["output"] = "\n".join(G._text(r, 20, 80) for _ in range(r.randint(50, max(60, target // 4000))))
            if it.get("type") == "reasoning":
                it["encrypted_content"] = G.base64.b64encode(r.randbytes(r.choice((2048, 6144, 12288)))).decode()
            items.append(it)
            size += len(json.dumps(it))
    req["input"] = items
    return json.dumps(req, ensure_ascii=r.random() < 0.4, separators=None if r.random() < 0.4 else (",", ":")).encode()


@functools.lru_cache(maxsize=None)
def realistic_corpus(n=18, lo=64 << 10, hi=8 << 20):
    """sizes spread log-uniformly between 64 KiB and 8 MiB (about 30 MB in all), every stream form"""
    r = random.Random(2024)
    out = []
    for i in range(n):
        target = int(2 ** r.uniform(16, 23))
        out.append(long_session(300 + i, max(lo, min(hi, target)), STREAM_FORMS[i % len(STREAM_FORMS)]))
    return tuple(out)


@functools.lru_cache(maxsize=None)
def verdict(body):
    """the oracle's ParseBody verdict of a body, computed once per test session: (verdict, model, stream)"""
    return Q.parse_body(body)


def expect(body, override="", prefix="v1", force=False):
    """Q.translate from the cached verdict: (verdict, path, body bytes or None, model, stream)"""
    v, model, stream = verdict(body)
    if v != Q.OK:
        return v, None, None, model, stream
    out = None
    if override:
        from _oracle import body_mutate
        rc, out = body_mutate(body, [], [("model", '"%s"' % override)])
        assert rc == 0
    elif force:
        out = body
    return v, Q.request_path(prefix), out, model, stream


# ================================================================ boundary bodies
EDGES = (THREAD, WARP, TILE, 2 * TILE, 3 * TILE)


def _placed(kind, at):
    """a body whose feature starts at byte `at`: the model value, a "type" tag value, a wrongly typed member value, or the root's
    closing brace; the bytes before it are an instructions string"""
    pre, post = {"model": (b'","model":', b'"gpt-5","input":"hi"}'),
                 "tag": (b'","input":[{"type":', b'"message","role":"user","content":"x"}]}'),
                 "type_error": (b'","max_output_tokens":', b'"5","input":"hi"}'),
                 "root": (b'","model":"m","input":"hi"', b"}")}[kind]
    head = b'{"instructions":"'
    n = at - len(head) - len(pre)
    if n < 0:
        return None
    body = head + b"a" * n + pre + post
    assert body[at:at + 1] == post[:1]
    return body


@functools.lru_cache(maxsize=None)
def boundary_bodies():
    """each feature within +-40 bytes of every thread, warp and tile boundary; bodies of 65535-65537 bytes"""
    out = []
    for kind in ("model", "tag", "type_error", "root"):
        for edge in EDGES:
            for delta in range(-40, 41, 4):
                b = _placed(kind, edge + delta)
                if b is not None:
                    out.append(b)
    head, tail = b'{"model":"m","stream":true,"input":[{"role":"user","content":"', b'"}]}'
    out += [head + b"a" * (n - len(head) - len(tail)) + tail for n in (65535, 65536, 65537, 65536 + TILE)]
    return tuple(out)


def deep(d):
    """nesting depth d under a member the request ignores"""
    v = "1"
    for _ in range(d - 1):
        v = '{"a":' + v + "}"
    return ('{"model":"m","input":"hi","x":' + v + "}").encode()


def near_16mib():
    """16 MiB - 1 bytes: a realistic session with a long function_call_output last"""
    body = long_session(9, 256 << 10)
    tail = b',{"type":"function_call_output","call_id":"c","output":"'
    k = (16 << 20) - 1 - (len(body) - 2) - len(tail) - len(b'"}]}')
    assert body.endswith(b"]}")
    return body[:-2] + tail + b"o" * k + b'"}]}'


def token_edge(k, length):
    """k one-byte scalars in an unknown member, padded to `length`: 2k + 12 scan tokens"""
    s = b'{"model":"m","x":[' + b",".join([b"1"] * k) + b"]}"
    return s + b" " * (length - len(s))


TOKEN_K = 3000
TOKEN_LEN = 4 * TOKEN_K - 2024   # 2k + 12 tokens == length / 2 + 1024


# ================================================================ malformed probes on the scan's boundaries
def _sites():
    """site -> (head, probe, post): the body is head + white space + probe + post"""
    return {
        "input_text": (b'{"model":"gpt-5","input":[{"type":"message","role":"user","content":[{"type":"input_text","text":"x"}]},',
                       b'{"role":"user","content":[{"type":"input_text","text":"q\\"r\\\\s\xc3\xa9 {}[]:, tru e"}]}', b']}'),
        "arguments": (b'{"model":"gpt-5","input":[{"type":"function_call","call_id":"c","name":"f","arguments":',
                      b'"{\\"a\\":[1,true,null],\\"s\\":\\"q\\\\\\"r\\"}"', b',"status":"completed"}]}'),
        "parameters": (b'{"model":"gpt-5","tools":[{"type":"function","name":"f","parameters":', D.PARAM_PROBE, b'}],"input":"hi"}'),
        "unknown": (b'{"model":"gpt-5","x_unknown":', D.PROBE, b',"input":"hi"}'),
    }


PROBE_BOUNDS = D.BOUNDS[:4]   # thread, warp, tile, second tile
PROBE_STRIDE = 8               # every eighth mutated body: the Python oracle reads about 1.6 MB/s


def probe_body(site, bound, k):
    head, probe, post = _sites()[site]
    body = head + D._pad(bound - k - len(head)) + probe + post
    assert body[bound] == probe[k]
    return body


@functools.lru_cache(maxsize=None)
def probe_corpus():
    """(label, bound, body) for every site, boundary and probe byte on it, with that byte deleted, duplicated or replaced"""
    out, seen = [], set()
    for site, (_, probe, _) in _sites().items():
        for kind, bound in PROBE_BOUNDS:
            for k in range(len(probe)):
                for name, m in D._mutations(probe_body(site, bound, k), bound):
                    if m not in seen:
                        seen.add(m)
                        out.append(("%s %s %d %s" % (site, kind, k, name), bound, m))
    return tuple(out[::PROBE_STRIDE])


def run_body(n, kind, where, twin):
    """n backslashes and a quote in an input text, the run starting on or ending at a boundary (test_large_scan_defects_cpu's
    run_body with this request's site)"""
    head, rest = b'{"model":"m","input":[{"role":"user","content":"', b'}]}'
    b = dict(D.BOUNDS[:3])[kind] if where == "start" else D._end_bound(kind, n)
    start = b if where == "start" else b - n
    closes = n % 2 == 0
    cont = b'a"' if closes != (twin == "valid") else b""
    return head + b"a" * (start - len(head)) + b"\\" * n + b'"' + cont + rest


@functools.lru_cache(maxsize=None)
def run_corpus():
    return tuple(("run%d %s %s %s" % (n, kind, where, twin), run_body(n, kind, where, twin))
                 for n in D.RUN_LENGTHS for kind in ("thread", "warp", "tile") for where in ("start", "end") for twin in ("valid", "malformed"))


def digest(bodies):
    h = hashlib.sha256()
    for b in bodies:
        h.update(len(b).to_bytes(8, "little")); h.update(b)
    return h.hexdigest()


# ================================================================ tests
DIGESTS = {
    "realistic": "dc4fff9b910e5580b954dc8641fd012cd6363dc127d1c999733d3eb631bea856",
    "boundary": "7ab18c7eabac260eb2fd7c512cd183ac4fdb024a836c6162464c52a9a9bce326",
    "probe": "89c4e11cbab7ba82b3ab6d722d74bd0afb9f99a8052975985a30d3ab4e3f1102",
    "run": "d8436b324ed3245dbafe7767b4aab5d7fc5996fddf423fde3bdd1fdc7d8b2fc4",
}


def test_corpus_shape_and_reproducible():
    c = realistic_corpus()
    # pinned: a change to the generator changes what the GPU tests compare, and shows here
    assert digest(c) == DIGESTS["realistic"]
    assert digest(boundary_bodies()) == DIGESTS["boundary"]
    assert digest(b for _, _, b in probe_corpus()) == DIGESTS["probe"]
    assert digest(b for _, b in run_corpus()) == DIGESTS["run"]
    sizes = [len(b) for b in c]
    assert min(sizes) >= 64 << 10 and max(sizes) <= 9 << 20 and max(sizes) >= 2 << 20, sizes
    assert 20 << 20 <= sum(sizes) <= 45 << 20, sum(sizes)
    kinds = b"".join(c)
    for needle in (b'"reasoning"', b'"encrypted_content"', b'"function_call_output"', b'"function_call"', b'"input_text"', b'"tools"'):
        assert needle in kinds, needle
    assert any(max(b) >= 0x80 for b in c) and any(max(b) < 0x80 for b in c)    # ensure_ascii off and on
    assert {b.startswith(b'{"model": ') for b in c} == {True, False}    # spaced and compact separators
    streams = {json.loads(b).get("stream", "absent") for b in c}
    assert streams == {"absent", False, True, None}, streams
    for b in c:   # a file-sized tool output and a multi-KB encrypted reasoning item in every session
        j = json.loads(b)
        assert max(len(i.get("output", "")) for i in j["input"]) > 2000
        assert max(len(i.get("encrypted_content", "")) for i in j["input"]) >= 2730


def test_oracle_accepts_realistic():
    for b in realistic_corpus():
        v, model, stream = verdict(b)
        j = json.loads(b)
        assert v == Q.OK and model == j["model"].encode() and stream == bool(j.get("stream")), len(b)


def test_boundary_shapes():
    bb = boundary_bodies()
    assert len(bb) > 300
    for kind in ("model", "tag", "type_error", "root"):
        for edge in EDGES[1:]:   # 32 is too close to the front for some of them
            b = _placed(kind, edge)
            assert verdict(b)[0] == (Q.FAIL if kind == "type_error" else Q.OK), (kind, edge)
    assert sorted(len(b) for b in bb)[-4:] == [65535, 65536, 65537, 65536 + TILE]


def test_limit_shapes():
    assert verdict(deep(48))[0] == Q.OK and json.loads(deep(49))
    big = near_16mib()
    assert len(big) == (16 << 20) - 1 and json.loads(big)["input"][-1]["type"] == "function_call_output"
    at, over = token_edge(TOKEN_K, TOKEN_LEN), token_edge(TOKEN_K + 1, TOKEN_LEN)
    assert len(at) == len(over) == TOKEN_LEN and json.loads(at) and json.loads(over)


def test_probe_corpus():
    """each probe byte sits on its boundary, and the corpus holds OKs and failures"""
    for site in _sites():
        for kind, bound in PROBE_BOUNDS:
            assert verdict(probe_body(site, bound, 0))[0] == Q.OK, (site, kind)
    pc = probe_corpus()
    assert len(pc) > 1000
    vs = [verdict(b)[0] for _, _, b in pc[::11]]
    assert vs.count(Q.OK) > 10 and vs.count(Q.FAIL) > 10
    rc = run_corpus()
    assert len(rc) == 120
    for label, b in rc:   # a valid twin is OK, a malformed one fails
        assert verdict(b)[0] == (Q.OK if label.endswith("valid") and not label.endswith("malformed") else Q.FAIL), label
