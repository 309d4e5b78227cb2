"""The Cohere /v2/rerank oracle (tests/_rerank_oracle.py) against the reference's own answers, and the corpora the GPU test
(test_rerank_gpu.py) feeds through every entry point: seeded request corpora (realistic RAG reranks and the decoder's edge rows),
buffered responses and raw error bodies.

Goldens: tests/golden/rerank_cases.json (lifted by extract_rerank_goldens.py)."""
import json
import math
import os
import random

import _rerank_oracle as Q
import test_translate_edges_cpu as E

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "rerank_cases.json"), encoding="utf-8"))
MAX_BODY = 65536   # the translate pass's largest size class


# ================================================================ realistic requests: RAG rerank calls
WORDS = ("password", "reset", "account", "the", "invoice", "refund", "Kubernetes", "pod", "restart", "policy", "naïve", "café", "東京",
         "データ", "señal", "Ελλάδα", "✓", "—", "𝔘𝔫𝔦𝔠𝔬𝔡𝔢", "\"quoted\"", "C:\\path", "line\nbreak", "tab\tstop", "emoji 🎉", "½")
MODELS = ("rerank-v3.5", "rerank-english-v3.0", "rerank-multilingual-v3.0", "rerank-english-v2.0", "BAAI/bge-reranker-v2-m3")
UNKNOWN = {"return_documents": lambda r: r.random() < 0.5, "rank_fields": lambda r: ["title", "text"], "max_chunks_per_doc": lambda r: r.randint(1, 10),
           "metadata": lambda r: {"trace": {"id": "%08x" % r.getrandbits(32), "tags": [1, None, "x"]}}, "user": lambda r: "u-%d" % r.randint(0, 99)}


def _text(r, lo, hi):
    n = int(min(hi, max(lo, r.lognormvariate(math.log(300), 0.9))))
    out = ""
    while len(out) < n:
        out += r.choice(WORDS) + " "
    return out[:n]


def realistic_request(seed):
    """One rerank call: a query and 1-200 retrieved chunks of 50-2000 characters, the optional ints, sometimes v1-style extras.
    json.dumps escapes the quotes, backslashes and control characters; a part is \\u-escaped ASCII-only JSON."""
    r = random.Random(seed)
    req = {"model": r.choice(MODELS), "query": _text(r, 5, 200)}
    ndocs = int(min(200, max(1, r.lognormvariate(math.log(15), 1.0))))
    req["documents"] = [_text(r, 50, 2000) for _ in range(ndocs)]
    if r.random() < 0.6:
        req["top_n"] = r.randint(1, max(1, ndocs))
    if r.random() < 0.3:
        req["max_tokens_per_doc"] = r.choice((512, 1024, 4096))
    if r.random() < 0.3:
        for k in r.sample(sorted(UNKNOWN), r.randint(1, 3)):
            req[k] = UNKNOWN[k](r)
    keys = list(req)
    r.shuffle(keys)
    req = {k: req[k] for k in keys}
    body = json.dumps(req, ensure_ascii=r.random() < 0.3, indent=2 if r.random() < 0.2 else None,
                      separators=None if r.random() < 0.5 else (",", ":")).encode()
    return body if len(body) <= MAX_BODY else realistic_request(seed + 7919)


def realistic_corpus(n=2000, seed=11):
    return [realistic_request(seed * 100003 + i) for i in range(n)]


# ================================================================ edge requests: every row of the decoder table at its boundary
BASE = {"model": "m", "query": "q", "documents": ["d"]}
MEMBERS = {"model": "rerank-v3.5", "query": "what", "documents": ["a", "b"], "top_n": 3, "max_tokens_per_doc": 512}
WRONG = [1, 1.5, "s", True, [], {}, [1], {"a": 1}, -0.0, ["a", 1], [None, {}]]
INTS = [b"0", b"-0", b"1", b"-5", b"9223372036854775807", b"9223372036854775808", b"-9223372036854775808", b"-9223372036854775809",
        b"99999999999999999999", b"1.0", b"1.5", b"1e2", b"1E0", b"-0.0", b"0e0", b'"3"', b"null", b"true"]
DOCS = [b"[]", b'["a",null]', b"[null]", b'["a",1]', b'["a",["b"]]', b'["a",{}]', b'[true]', b'"a"', b"{}", b"null",
        b'["\\u00e9\\n\\"x\\""]', b'["a\\/b"]']


def _dump(o):
    return json.dumps(o, separators=(",", ":")).encode()


def _with(member, raw):
    return b'{"model":"m","query":"q","%s":%s}' % (member.encode(), raw) if member != "model" else b'{"%s":%s,"query":"q"}' % (member.encode(), raw)


def edge_corpus():
    out = []
    for k, v in MEMBERS.items():
        out.append(_dump(dict(BASE, **{k: v})))
        out.append(_dump(dict(BASE, **{k: None})))
        out.append(_dump(dict(BASE, **{k: v, "unknown_" + k: {"x": [1, None, {"y": [[]]}]}})))
        for w in WRONG:
            out.append(_dump(dict(BASE, **{k: w})))
        b = _dump(dict(BASE, **{k: v}))   # the member twice
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(v)))
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(WRONG[0])))
    for k in ("top_n", "max_tokens_per_doc"):
        out += [_with(k, x) for x in INTS]
    out += [_with("documents", x) for x in DOCS]
    out += [b"null", b" null ", b"[]", b'"s"', b"{}", b"1", b" {} ", b'{"model":"m"} x', b'{"model":"m",}', b'{"query":"a\x01b"}',
            b'{"mod\\u0065l":"m"}', b'{"model":"m\\u0065"}', b'{"model":"m\\/x"}', b'{"Model":5,"Query":1,"DOCUMENTS":"x"}',
            b'{"model":null,"query":null,"documents":null,"top_n":null,"max_tokens_per_doc":null}', b'{"model":"m","top_n":"x","query":5}',
            b'{"model":"m","query":5,"top_n":"x"}', b'{"model":"m","return_documents":true,"rank_fields":["a"]}',
            b'{"model":"m","x":' + b"[" * 47 + b"]" * 47 + b"}", b'{"model":"m","x":' + b"[" * 48 + b"]" * 48 + b"}",
            b'{"model":"m","documents":["\xff\xfe"]}', b'{"model":"m","top_n":-5}', b'{"model":"m","query":"q","documents":["a"]}   ']
    return out


def class_bound_bodies():
    """bodies of exactly c-1, c and c+1 bytes for every size class bound, and one over 64 KiB"""
    out = []
    for c in E.CLASSES:
        for n in (c - 1, c, c + 1):
            head, tail = b'{"model":"m","query":"q","documents":["', b'"],"top_n":1}'
            out.append(head + b"a" * (n - len(head) - len(tail)) + tail)
    return out


# ================================================================ documents at the index stage's token capacity
def docs_body(k, length):
    """k one-character documents (two index tokens each: the string and its comma), padded to `length` bytes by the query"""
    docs = b",".join(b'"%c"' % (97 + j % 26) for j in range(k))
    head, mid = b'{"model":"m","query":"', b'","documents":[%s]}' % docs
    pad = length - len(head) - len(mid)
    assert pad >= 0, (k, length)
    return head + b"x" * pad + mid


def capacity_cases(ktok=None, classes=None):
    """(class, k, body with k documents, body with k+1): k is the most documents whose body fits the class's token capacity;
    both bodies have the same length, 64 bytes below the class bound"""
    ktok = ktok or E.KTOK
    out = []
    for c in classes or E.CLASSES:
        n = c - 64
        k = 1
        while E.count_tokens(docs_body(k + 1, n)) <= ktok[c]:
            k += 1
        out.append((c, k, docs_body(k, n), docs_body(k + 1, n)))
    return out


# ================================================================ buffered responses
def _score(r):
    """relevance scores as the API prints them; now and then one in exponent form, which declines (its range is not restated)"""
    if r.random() < 0.005:
        return 1e-5
    return r.choice((lambda: round(r.uniform(0.001, 1), 8), lambda: r.uniform(0.001, 1), lambda: 0, lambda: 1))()


def realistic_response(seed):
    r = random.Random(seed)
    n = r.randint(0, 50)
    resp = {"results": [{"index": r.randint(0, 200), "relevance_score": _score(r)} for _ in range(n)], "id": "%08x-%04x" % (r.getrandbits(32), r.getrandbits(16))}
    if r.random() < 0.9:
        meta = {"api_version": {"version": r.choice(("2", "1")), "is_experimental": r.random() < 0.2}}
        if r.random() < 0.3:
            meta["api_version"]["is_deprecated"] = False
        meta["billed_units"] = {"search_units": r.choice((1, 1.0, 2))}
        if r.random() < 0.85:
            tok = {"input_tokens": r.choice((r.randint(0, 200000), float(r.randint(0, 200000)), r.randint(0, 5000) + r.choice((0.25, 0.5, 0.75))))}
            if r.random() < 0.3:
                tok["output_tokens"] = r.randint(0, 100)
            meta["tokens"] = tok
        if r.random() < 0.1:
            meta["warnings"] = ["model deprecated", "x"]
        if r.random() < 0.1:
            meta["cached_tokens"] = r.randint(0, 1000)
        resp["meta"] = meta
    if r.random() < 0.1:
        resp["model"] = "rerank-v3.5"   # not a RerankV2Response member: skipped
    return json.dumps(resp, indent=2 if r.random() < 0.3 else None).encode()


# float texts around the integer boundaries of the uint32(float64) conversion
FLOAT_TEXTS = [b"0", b"-0", b"0.0", b"-0.0", b"-0.5", b"-0.99999999999999994", b"-0.99999999999999995", b"-0.9999999999999999999", b"-1", b"-1.0",
               b"0.99999999999999994", b"0.99999999999999995", b"0.999999999999999944488848768742172978818416595458984375",
               b"0.99999999999999994448884876874217297881841659545898437", b"0.9999999999999999444888487687421729788184165954589843751",
               b"1", b"1.5", b"24.99999999999999999", b"24.999999999999996", b"24.9999999999999964", b"2.9999999999999996",
               b"2.99999999999999977795539507496869191527366638183593750", b"2.99999999999999977795539507496869191527366638183593749",
               b"4294967295", b"4294967295.0", b"4294967295.4", b"4294967295.99999", b"4294967295.9999995", b"4294967295.99999952316",
               b"4294967295.999999523162841796875", b"4294967295.999999523162841796874", b"4294967296", b"4294967296.0", b"18446744073709551616",
               b"2147483647.5", b"2147483648", b"1e2", b"1E0", b"2.5e-3", b"1" * 308, b"1" * 309, b"0." + b"9" * 400, b"7." + b"0" * 300 + b"1",
               b"16777216.999999999", b"9007199254740993", b"12345678901", b"00", b"1.", b"-", b'"5"', b"true", b"null"]


def token_response(inp, out=b"null", extra=b""):
    return b'{"results":[{"index":0,"relevance_score":0.5}],"meta":{"tokens":{"input_tokens":%s,"output_tokens":%s}%s}}' % (inp, out, extra)


def edge_responses():
    out = [g["body"].encode() for g in GOLD["response_body"]]
    for t in FLOAT_TEXTS:
        out += [token_response(t), token_response(b"1", t), token_response(t, t)]
        out.append(b'{"results":[{"index":0,"relevance_score":%s}]}' % t)
        out.append(b'{"meta":{"cached_tokens":%s,"billed_units":{"images":%s}}}' % (t, t))
    out += [token_response(b"4294967295", b"1"), token_response(b"4294967295", b"4294967295"), token_response(b"3000000000", b"3000000000.7")]
    wrong = [b"1", b"1.5", b'"s"', b"true", b"[]", b"{}", b"[1]", b"[null]", b"null"]
    for w in wrong:
        out += [b'{"results":%s}' % w, b'{"results":[%s]}' % w, b'{"id":%s}' % w, b'{"meta":%s}' % w, b'{"results":[{"index":%s}]}' % w,
                b'{"meta":{"api_version":%s}}' % w, b'{"meta":{"api_version":{"version":%s,"is_deprecated":%s}}}' % (w, w),
                b'{"meta":{"billed_units":%s}}' % w, b'{"meta":{"tokens":%s}}' % w, b'{"meta":{"warnings":%s}}' % w,
                b'{"meta":{"warnings":[%s]}}' % w, b'{"meta":{"api_version":{"is_experimental":%s}}}' % w]
    out += [b"", b"   ", b"null", b" null x", b"{}", b"[]", b'"x"', b"1", b'{"results":[]} trailing', b'{"results":[]}{', b'{"results":[',
            b'{"meta":{"tokens":{}}}', b'{"meta":{"tokens":null}}', b'{"meta":{"tokens":{"input_tokens":null,"output_tokens":null}}}',
            b'{"meta":{"tokens":{"input_tokens":1},"tokens":{"input_tokens":2}}}', b'{"meta":{"tokens":{"input_tokens":1,"input_tokens":2}}}',
            b'{"meta":{"tok\\u0065ns":{"input_tokens":1}}}', b'{"id":"a\\u0041\\n"}', b'{"results":[null,{"index":1,"relevance_score":null}]}',
            b'{"results":[{"index":1,"x":{"deep":[[[{}]]]}}],"unknown":[1,{"a":null}]}', b'{"Meta":{"tokens":{"input_tokens":7}}}',
            b'{"meta":{"tokens":{"input_tokens":7,"extra":1.5e999}}}', b'{"meta":{"tokens":{"Input_Tokens":7}}}',
            b'{"results":[{"index":1.0}]}', b'{"results":[{"index":9223372036854775808}]}', b'{"results":[{"index":-9223372036854775808}]}',
            b'{"x":' + b"[" * 70 + b"]" * 70 + b"}", b'{"meta":{"tokens":{"input_tokens":5}}}\x00\xff']
    return out


def response_corpus(n=2000, seed=17):
    return [realistic_response(seed * 100003 + i) for i in range(n)] + edge_responses()


# ================================================================ raw error bodies
def error_bodies():
    r = random.Random(23)
    out = [g["body"].encode() for g in GOLD["response_error"]]
    out += [b"", b"x", b'"', b"\\", b'say "hi"\n', b"\x00\x01\x1f\x7f", b"<html><body>502 Bad Gateway</body></html>", b"caf\xc3\xa9",
            b"\t\r\n", b"a" * 3000, b"upstream connect error or disconnect/reset before headers. reset reason: overflow", b"{not json"]
    for _ in range(300):
        out.append(bytes(r.choice(b'abc "\\\n\t\x01<>&{}') for _ in range(r.randint(1, 200))))
    return out


# ================================================================ tests
def test_request_body_goldens():
    for c in GOLD["request_body"]:
        v, path, out, model = Q.translate(c["body"].encode(), c["override"], c["version"], c["force"])
        assert v == Q.OK and path == c["exp_path"] and model == b"rerank-english-v3", c["name"]
        if c["exp_body_contains"]:
            assert c["exp_body_contains"].encode() in out, c["name"]
            assert json.loads(out)["model"] == c["override"]
        else:
            assert out == (c["body"].encode() if c["force"] else None), c["name"]


def test_parse_body_goldens():
    for c in GOLD["parse_body"]:
        v, model = Q.parse_body(c["body"].encode())
        assert (v, model.decode()) == ((Q.FAIL, "") if c["error"] else (Q.OK, c["model"])), c["name"]


def test_response_goldens():
    for c in GOLD["response_body"]:
        v, u = Q.response_usage(c["body"].encode())
        if c["error"]:
            assert v == Q.FAIL, c["name"]
        else:
            assert (v, u) == (Q.OK, (c["input"], c["output"], c["total"])), c["name"]


def test_error_goldens():
    for c in GOLD["response_error"]:
        v, out = Q.response_error(c["body"].encode(), "json" not in c["content_type"])
        assert v == Q.OK
        if c["passthrough"]:
            assert out is None
        else:
            assert json.loads(out) == {"message": c["body"]}


def test_oracle_known_answers():
    cases = {
        b'{"model":"m","query":"q","documents":["a",null]}': Q.OK, b'{"documents":null}': Q.OK, b'{"documents":[]}': Q.OK,
        b'{"documents":["a",1]}': Q.FAIL, b'{"documents":"a"}': Q.FAIL, b'{"top_n":-5}': Q.OK, b'{"top_n":1.0}': Q.FAIL, b'{"top_n":1e2}': Q.FAIL,
        b'{"top_n":9223372036854775807}': Q.OK, b'{"top_n":9223372036854775808}': Q.FAIL, b'{"max_tokens_per_doc":"1"}': Q.FAIL,
        b'{"model":5}': Q.FAIL, b'{"query":[]}': Q.FAIL, b'{"model":"m","model":"n"}': Q.OUT, b'{"model":"m\\u0065"}': Q.OUT,
        b'{"qu\\u0065ry":"m"}': Q.OUT, b'{"return_documents":true,"rank_fields":["x"]}': Q.OK, b'{"Model":1}': Q.OK, b"null": Q.OUT,
        b"[]": Q.FAIL, b'"x"': Q.FAIL, b'{"model":"m"}x': Q.FAIL, b'{"model":"m","top_n":"x","query":5}': Q.FAIL, b"{": Q.FAIL,
        b'{"model":"m","query":5,"model":"n"}': Q.FAIL, b'{"model":"m","model":"n","query":5}': Q.OUT,
    }
    for body, exp in cases.items():
        assert Q.parse_body(body)[0] == exp, body
    assert Q.request_path("v2") == "/v2/rerank" and Q.request_path("") == "/rerank" and Q.request_path("/a//b/./c/") == "/a/b/c/rerank"
    assert Q.request_path("v2/..") == "/rerank" and Q.request_path("../../x") == "/x/rerank" and Q.request_path("a/../b/..") == "/rerank"
    v, path, out, _ = Q.translate(b' {"query":"x"} ', "o-1")
    assert (v, out) == (Q.OK, b'{"query":"x","model":"o-1"}')   # sjson appends at the root and drops the bytes outside it
    usage = {
        token_response(b"24.99999999999999999"): (25, -1, 25), token_response(b"24.999999999999996"): (24, -1, 24),
        token_response(b"0.99999999999999995"): (1, -1, 1), token_response(b"0.99999999999999994"): (0, -1, 0),
        token_response(b"-0.5"): (0, -1, 0), token_response(b"4294967295.4", b"1"): (4294967295, 1, 0),
        token_response(b"4294967295.9999995"): (4294967295, -1, 4294967295), token_response(b"4294967295.99999988"): None, token_response(b"-1"): None, token_response(b"1e2"): None,
        b'{"meta":{"tokens":{}}}': (-1, -1, 0), b'{"meta":{"tokens":null}}': (-1, -1, -1), b'{"meta":null}': (-1, -1, -1),
    }
    for body, exp in usage.items():
        v, u = Q.response_usage(body)
        assert (v, u) == ((Q.OUT, None) if exp is None else (Q.OK, exp)), body
    assert Q.response_usage(b"")[0] == Q.FAIL and Q.response_usage(b'{"results":[]} x')[0] == Q.OK and Q.response_usage(b'{"id":1}')[0] == Q.FAIL
    assert Q.response_error(b'a"\n\x01', True) == (Q.OK, b'{"message":"a\\"\\n\\u0001"}')
    assert Q.response_error(b"", True) == (Q.OUT, b'{"message":""}') and Q.response_error(b"x", False) == (Q.OK, None)


def test_corpus_generators():
    bodies = realistic_corpus(2000)
    assert len(set(bodies)) == len(bodies) and all(len(b) <= MAX_BODY for b in bodies)
    assert all(Q.parse_body(b)[0] == Q.OK for b in bodies)
    ndocs = [len(json.loads(b)["documents"]) for b in bodies]
    assert min(ndocs) == 1 and max(ndocs) >= 100
    joined = b"".join(bodies)
    for needle in (b"\\n", b'\\"', b"\\u", b'"top_n"', b'"max_tokens_per_doc"', b'"return_documents"', "東京".encode()):
        assert needle in joined, needle
    verdicts = [Q.parse_body(b)[0] for b in edge_corpus()]
    assert {Q.OK, Q.FAIL, Q.OUT} <= set(verdicts)
    resp = response_corpus()
    assert len(resp) >= 2000
    rv = [Q.response_usage(b)[0] for b in resp]
    assert {Q.OK, Q.FAIL, Q.OUT} <= set(rv)
    for c, k, fit, over in capacity_cases():
        assert len(fit) == len(over) and E.count_tokens(fit) <= E.KTOK[c] < E.count_tokens(over), c
        assert Q.parse_body(fit)[0] == Q.OK and Q.parse_body(over)[0] == Q.OK
