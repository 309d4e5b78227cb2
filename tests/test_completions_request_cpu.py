"""The /v1/completions request oracle (tests/_completions_request_oracle.py) against the reference's own answers, and the corpus
generators the GPU test (test_completions_request_gpu.py) feeds through every entry point.

Goldens: tests/golden/completions_request_cases.json (lifted by extract_completions_request_goldens.py): the prompt-union cases,
the ParseBody and RequestBody cases of the reference's tests, and the request bodies of its nine recorded completion cassettes."""
import json
import math
import os
import random

import _completions_request_oracle as Q
import test_translate_edges_cpu as E

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = json.load(open(os.path.join(HERE, "golden", "completions_request_cases.json"), encoding="utf-8"))
MAX_BODY = 65536   # the translate pass's largest size class


# ================================================================ realistic corpus: code completion and vLLM clients
CODE = ("def fib(n):\n    if n <= 1:\n        return n\n    return fib(n - 1) + fib(n - 2)\n", "import numpy as np\n",
        "for (int i = 0; i < n; i++) {\n    sum += a[i] * b[i];\n}\n", "    # TODO: handle the \"empty\" case\\n here\n",
        "SELECT id, name FROM users WHERE created_at > '2024-01-01';\n", "fn main() {\n    println!(\"héllo, wörld — ✓\");\n}\n",
        "class Cache:\n    def __init__(self):\n        self.d = {}\n", "\t// 日本語のコメント\n\treturn nil\n")
MODELS = ("babbage-002", "gpt-3.5-turbo-instruct", "qwen2.5-coder-7b", "deepseek-coder-6.7b-base", "starcoder2-15b",
          "meta-llama/Llama-3.1-8B", "codellama-lora-sql")
VLLM = {   # sampling keys vLLM accepts that openai.CompletionRequest does not have: skipped by the decoder
    "top_k": lambda r: r.choice((-1, 20, 40)), "min_p": lambda r: round(r.random() * 0.2, 3), "repetition_penalty": lambda r: round(1 + r.random() * 0.3, 2),
    "guided_json": lambda r: {"type": "object", "properties": {"name": {"type": "string"}, "tags": {"type": "array", "items": {"type": "string"}}}, "required": ["name"]},
    "guided_choice": lambda r: ["yes", "no"], "guided_regex": lambda r: "[0-9]{3}-[0-9]{4}", "skip_special_tokens": lambda r: r.random() < 0.5,
    "stop_token_ids": lambda r: [r.randint(0, 50000) for _ in range(r.randint(1, 4))], "include_stop_str_in_output": lambda r: False,
    "min_tokens": lambda r: r.randint(0, 8), "ignore_eos": lambda r: False, "prompt_logprobs": lambda r: None,
    "lora_request": lambda r: {"lora_name": "sql-adapter", "lora_int_id": 1, "lora_path": "/adapters/sql"},
}
STOPS = (lambda r: "\n\n", lambda r: ["\n\n", "\ndef ", "</s>"], lambda r: [], lambda r: None, lambda r: {"weird": [1, {"x": None}]},
         lambda r: 3, lambda r: True)


def _code(r, median, hi):
    """source text of a log-normal length (at most hi characters)"""
    n = int(min(hi, r.lognormvariate(math.log(median), 1.2)))
    out = ""
    while len(out) < n:
        out += r.choice(CODE)
    return out[:n]


def _ids(r, n):
    return [r.randint(0, 100_000) for _ in range(n)]


def realistic_request(seed):
    """One completion request: fill-in-the-middle, plain string, string batch, token ids or token-id batch, with the sampling
    parameters these clients send; a third carry vLLM extras.  About a quarter is pretty-printed."""
    r = random.Random(seed)
    kind = r.choices(("fim", "string", "batch", "tokens", "token_batch"), (5, 4, 2, 2, 1))[0]
    req = {"model": r.choice(MODELS)}
    if kind == "fim":
        req["prompt"] = _code(r, 1500, 30000)
        req["suffix"] = _code(r, 300, 8000)
    elif kind == "string":
        req["prompt"] = _code(r, 2000, 60000)
    elif kind == "batch":
        req["prompt"] = [_code(r, 600, 8000) for _ in range(r.randint(1, 8))]
    elif kind == "tokens":
        req["prompt"] = _ids(r, int(min(3000, r.lognormvariate(4, 1.0))))
    else:
        req["prompt"] = [_ids(r, int(min(600, r.lognormvariate(3.5, 0.8)))) for _ in range(r.randint(1, 4))]
    req["max_tokens"] = r.choice((16, 64, 256, 1024))
    if r.random() < 0.6:
        req["temperature"] = r.choice((0, 0.2, 0.7, 1.0, 1.25))
    if r.random() < 0.4:
        req["top_p"] = r.choice((0.9, 0.95, 1))
    if r.random() < 0.5:
        req["stop"] = r.choice(STOPS)(r)
    if r.random() < 0.2:
        req["n"] = r.randint(1, 4)
    if r.random() < 0.1:
        req["best_of"] = req.get("n", 1) + 1
    if r.random() < 0.15:
        req["logprobs"] = r.randint(0, 5)
    if r.random() < 0.1:
        req["echo"] = r.random() < 0.5
    if r.random() < 0.15:
        req["seed"] = r.randint(-(1 << 63), (1 << 63) - 1)
    if r.random() < 0.1:
        req["logit_bias"] = {str(r.randint(0, 50000)): r.randint(-100, 100) for _ in range(r.randint(1, 5))}
    if r.random() < 0.2:
        req["frequency_penalty"] = round(r.uniform(-2, 2), 2)
        req["presence_penalty"] = round(r.uniform(-2, 2), 2)
    if r.random() < 0.1:
        req["user"] = "user-%06d" % r.randint(0, 999999)
    req["stream"] = r.random() < 0.6
    if req["stream"] and r.random() < 0.5:
        req["stream_options"] = {"include_usage": True}
    if r.random() < 0.35:
        for k in r.sample(sorted(VLLM), r.randint(1, 5)):
            req[k] = VLLM[k](r)
    keys = list(req)
    r.shuffle(keys)
    req = {k: req[k] for k in keys}
    body = json.dumps(req, ensure_ascii=r.random() < 0.3, indent=2 if r.random() < 0.25 else None,
                      separators=None if r.random() < 0.5 else (",", ":")).encode()
    return body if len(body) <= MAX_BODY else realistic_request(seed + 7919)


def realistic_corpus(n=2000, seed=5):
    return [realistic_request(seed * 100003 + i) for i in range(n)]


# ================================================================ edge corpus: every row of the decoder table at its boundary
BASE = {"model": "m", "prompt": "p"}
MEMBERS = {"model": "gpt", "suffix": "s", "user": "u", "best_of": 2, "logprobs": 1, "max_tokens": 5, "n": 1, "seed": 7,
           "frequency_penalty": 0.5, "presence_penalty": -1, "temperature": 1, "top_p": 0.9, "echo": True, "stream": True,
           "logit_bias": {"50256": -100}, "stop": ["\n"], "stream_options": {"include_usage": True}, "prompt": [1, 2]}
WRONG = [1, 1.5, "s", True, [], {}, [1], {"a": 1}, -0.0]
INTS = [b"0", b"-0", b"1", b"-1", b"9223372036854775807", b"9223372036854775808", b"-9223372036854775808", b"-9223372036854775809",
        b"999999999999999999", b"1000000000000000000", b"99999999999999999999", b"1.0", b"1.5", b"1e2", b"1E0", b"-0.0", b"0e0"]
FLOATS = [b"0", b"-0", b"0.5", b"-0.0", b"1e308", b"1e309", b"1E-5", b"2.5e0", b"1" * 308, b"1" * 309, b"-" + b"9" * 308,
          b"1.7976931348623157", b"0." + b"0" * 400 + b"1", b"3"]
PROMPTS = [b'""', b'"x"', b'[]', b'[ ]', b'["a"]', b'["a",null]', b'["a",1]', b'["a",["b"]]', b'[null]', b'[null,"a"]', b'[{}]', b'[true]',
           b'[false,1]', b'[1]', b'[-1,0,null]', b'[1,"a"]', b'[1,1.5]', b'[1,1e2]', b'[1,[2]]', b'[9223372036854775807]',
           b'[9223372036854775808]', b'[-9223372036854775808]', b'[-9223372036854775809]', b'[[]]', b'[[1],null,[null,2]]',
           b'[[1],[2,"x"]]', b'[[1],3]', b'[[1],[1.0]]', b'[[-9223372036854775809]]', b'[[9223372036854775807,0]]', b'null', b'1', b'true',
           b'{}', b'{"a":1}', b'"a\\u0000b"', b'"\\/path"', b'[[1],[2]] ', b' "x"', b'[ -1 , 2 ]']
STOP_FORMS = [b'"x"', b'["a","b"]', b'[]', b'null', b'1', b'1e999', b'true', b'{"a":[{"b":null}]}', b'[1,"a",null,{}]']


def _dump(o):
    return json.dumps(o, separators=(",", ":")).encode()


def _with(member, raw):
    return b'{"model":"m","prompt":"p","%s":%s}' % (member.encode(), raw) if member not in ("model", "prompt") else \
        b'{"%s":%s,"x":1}' % (member.encode(), raw)


def edge_corpus():
    out = []
    for k, v in MEMBERS.items():
        out.append(_dump(dict(BASE, **{k: v})))
        out.append(_dump(dict(BASE, **{k: None})))
        out.append(_dump(dict(BASE, **{k: v, "unknown_" + k: {"x": [1, None]}})))
        for w in WRONG:
            out.append(_dump(dict(BASE, **{k: w})))
        b = _dump(dict(BASE, **{k: v}))   # the member twice
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(v)))
        out.append(b[:-1] + b',"%s":%s}' % (k.encode(), _dump(WRONG[0])))
    for k in ("best_of", "logprobs", "max_tokens", "n", "seed"):
        out += [_with(k, x) for x in INTS]
        out += [_with("logit_bias", b'{"1":%s}' % x) for x in INTS[4:8]]
    for k in ("frequency_penalty", "presence_penalty", "temperature", "top_p"):
        out += [_with(k, x) for x in FLOATS]
    out += [_with("prompt", x) for x in PROMPTS]
    out += [_with("stop", x) for x in STOP_FORMS]
    out += [b'{"model":"m","logit_bias":{"1":1,"1":2}}', b'{"model":"m","logit_bias":{"a\\u0062":1}}', b'{"model":"m","logit_bias":{"1":null}}',
            b'{"model":"m","logit_bias":{"1":"1"}}', b'{"model":"m","logit_bias":[]}', b'{"model":"m","logit_bias":{"1":1.5}}',
            b'{"model":"m","stream_options":{"include_usage":null}}', b'{"model":"m","stream_options":{"include_usage":1}}',
            b'{"model":"m","stream_options":{"include_usage":true,"include_usage":false}}', b'{"model":"m","stream_options":{"x":[1],"continuous_usage_stats":true}}',
            b'{"model":"m","stream_options":{"incl\\u0075de_usage":true}}', b'{"model":"m","stream_options":[]}', b'{"model":"m","include_usage":"x"}',
            b'{"mod\\u0065l":"m"}', b'{"model":"m\\u0065"}', b'{"model":"m\\/x","prompt":"p"}', b'{"Model":5,"Prompt":null,"STREAM":"x"}', b'{"model":"m","prompt":"p","stream":true,"Stream":1}',
            b'null', b' null ', b'[]', b'"s"', b'{}', b'1', b' {"model":"m"} ', b'{"model":"m"} x', b'{"model":"m",}', b'{"prompt":"a\x01b"}',
            b'{"model":null,"prompt":null}', b'{"model":"m","prompt":null,"max_tokens":"x"}', b'{"model":"m","max_tokens":"x","prompt":null}',
            b'{"model":"m","temperature":1e400,"max_tokens":"x"}', b'{"model":"m","max_tokens":"x","temperature":1e400}',
            b'{"model":"m","prompt":[[' + b"[" * 50 + b"]" * 50 + b']]}', b'{"model":"m","x":' + b"[" * 47 + b"]" * 47 + b'}',
            b'{"model":"m","x":' + b"[" * 48 + b"]" * 48 + b'}', b'{"model":"m","max_tokens":-1,"temperature":3,"prompt":""}']
    return out


def class_bound_bodies():
    """bodies of exactly c-1, c and c+1 bytes for every size class bound, and one over 64 KiB"""
    out = []
    for c in E.CLASSES:
        for n in (c - 1, c, c + 1):
            head, tail = b'{"model":"m","stream":true,"prompt":"', b'","suffix":"\\n"}'
            out.append(head + b"a" * (n - len(head) - len(tail)) + tail)
    return out


# ================================================================ token-id prompts at the index stage's capacity
def token_prompt_body(k, length):
    """a compact token-id prompt of k five-digit ids, padded to `length` bytes by the suffix string (two tokens whatever its length)"""
    ids = b",".join(b"%d" % (10000 + (j * 7919) % 90000) for j in range(k))
    head, mid = b'{"model":"m","suffix":"', b'","prompt":[%s]}' % ids
    pad = length - len(head) - len(mid)
    assert pad >= 0, (k, length)
    return head + b"x" * pad + mid


def capacity_cases(ktok=None, classes=None):
    """(class, k, body with k ids, body with k+1 ids): k is the most ids whose body fits the class's token capacity (ktok[c]);
    both bodies have the same length, 64 bytes below the class bound"""
    ktok = ktok or E.KTOK
    out = []
    for c in classes or E.CLASSES:
        n = c - 64
        fixed = E.count_tokens(token_prompt_body(1, n)) - 1   # each further id adds a comma and a scalar
        k = (ktok[c] - fixed + 1) // 2   # k ids: fixed + 2k - 1 tokens
        out.append((c, k, token_prompt_body(k, n), token_prompt_body(k + 1, n)))
    return out


# ================================================================ mutants
MUTATION_SEEDS = 40


def mutation_seeds():
    r = random.Random(13)
    gold = [c["body"].encode() for c in GOLD["cassettes"] + GOLD["request_body"]] + [u["wrapped"].encode() for u in GOLD["unions"]]
    small = [b for b in realistic_corpus(400, seed=3) if len(b) < 900]
    seeds = sorted(set(gold), key=gold.index)
    return seeds + r.sample(small, max(0, min(len(small), MUTATION_SEEDS - len(seeds))))


# ================================================================ tests
def test_union_goldens():
    """each unmarshalJSONNestedUnion case as the prompt of a request: what the reference decodes is OK; what it rejects fails,
    except a null prompt, which is outside the subset"""
    assert len(GOLD["unions"]) >= 20
    for u in GOLD["unions"]:
        v, model, _ = Q.parse_body(u["wrapped"].encode())
        want = Q.FAIL if u["error"] else Q.OK
        if u["json"] == "null":
            want = Q.OUT
        assert v == want, (u["test"], u["name"], v)
        if v == Q.OK:
            assert model == b"m"


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
            assert b'"model":"%s"' % c["exp_model_member"].encode() in out
        else:
            assert out == (None if c["exp_body"] is None else c["body"].encode()), c["name"]


def test_cassette_requests():
    """every recorded request decodes, the bad-request one included (the decoder checks no ranges)"""
    assert len(GOLD["cassettes"]) == 9
    for c in GOLD["cassettes"]:
        body = c["body"].encode()
        assert len(body) == c["content_length"]
        v, path, out, model, stream = Q.translate(body)
        want = json.loads(body)
        assert (v, path, out, model.decode(), stream) == (Q.OK, "/v1/completions", None, want["model"], want.get("stream", False)), c["name"]
    forms = {c["name"]: type(json.loads(c["body"])["prompt"]).__name__ for c in GOLD["cassettes"]}
    assert forms["completion-token"] == "list" and forms["completion-token-batch"] == "list" and forms["completion-basic"] == "str"


def test_oracle_known_answers():
    cases = {
        b'{"model":"m","prompt":"x"}': Q.OK, b'{"model":"m","prompt":[]}': Q.OK, b'{"model":"m","prompt":["a",null]}': Q.OK,
        b'{"model":"m","prompt":[[1],null,[null,2]]}': Q.OK, b'{"model":"m","prompt":[-1,null,3]}': Q.OK,
        b'{"model":"m","prompt":[null,"a"]}': Q.FAIL, b'{"model":"m","prompt":[true]}': Q.FAIL, b'{"model":"m","prompt":[1,"a"]}': Q.FAIL,
        b'{"model":"m","prompt":[[1],2]}': Q.FAIL, b'{"model":"m","prompt":{}}': Q.FAIL, b'{"model":"m","prompt":null}': Q.OUT,
        b'{"model":"m","prompt":[9223372036854775807,-9223372036854775808]}': Q.OK, b'{"model":"m","prompt":[9223372036854775808]}': Q.FAIL,
        b'{"model":"m","prompt":[[-9223372036854775809]]}': Q.FAIL, b'{"model":"m","max_tokens":1.0}': Q.FAIL,
        b'{"model":"m","max_tokens":1e2}': Q.FAIL, b'{"model":"m","max_tokens":-0}': Q.OK, b'{"model":"m","seed":9223372036854775807}': Q.OK,
        b'{"model":"m","seed":-9223372036854775809}': Q.FAIL, b'{"model":"m","temperature":1e2}': Q.OUT,
        b'{"model":"m","temperature":' + b"9" * 308 + b'}': Q.OK, b'{"model":"m","temperature":' + b"9" * 309 + b'}': Q.OUT,
        b'{"model":"m","temperature":"1"}': Q.FAIL, b'{"model":"m","logit_bias":{"1":2,"1":null}}': Q.OK,
        b'{"model":"m","logit_bias":{"1":2.5}}': Q.FAIL, b'{"model":"m","stop":{"a":[1e999]}}': Q.OUT, b'{"model":"m","stop":[1,"1e999",-2.5,' + b"9" * 308 + b']}': Q.OK,
        b'{"model":"m","stream_options":{"include_usage":"y"}}': Q.FAIL, b'{"model":"m","stream_options":{"other":"y"}}': Q.OK,
        b'{"model":"m","Prompt":5,"STREAM":"x"}': Q.OK, b'{"model":"m","model":"n"}': Q.OUT, b'{"model":5}': Q.FAIL,
        b'{"model":"m\\u0065"}': Q.OUT, b'{"mod\\u0065l":"m"}': Q.OUT, b'{"model":"m","prompt":null,"n":"x"}': Q.OUT,
        b'{"model":"m","n":"x","prompt":null}': Q.FAIL, b'null': Q.OUT, b'[]': Q.FAIL, b'{"model":"m"}x': Q.FAIL,
        b'{"model":"m","include_usage":5}': Q.OK, b'{"model":"m","stream_options":{"include_usage":true,"include_usage":true}}': Q.OUT,
    }
    for body, exp in cases.items():
        assert Q.parse_body(body)[0] == exp, body
    assert Q.parse_body(b'{"model":"m","stream":true}')[1:] == (b"m", True)
    assert Q.request_path("") == "/completions" and Q.request_path("/custom/api/") == "/custom/api/completions"
    v, path, out, _, _ = Q.translate(b' {"prompt":"x"} ', "o-1")
    assert (v, out) == (Q.OK, b'{"prompt":"x","model":"o-1"}')   # sjson appends at the root and drops the bytes outside it
    v, path, out, _, _ = Q.translate(b'{"model": null, "prompt":"x"}', "o-1")
    assert out == b'{"model": "o-1", "prompt":"x"}'


def test_realistic_corpus_generator():
    bodies = realistic_corpus(2000)
    assert len(set(bodies)) == len(bodies)
    assert all(len(b) <= MAX_BODY for b in bodies)
    assert all(Q.parse_body(b)[0] == Q.OK for b in bodies)
    assert {E.class_of(len(b)) for b in bodies} == set(E.CLASSES)   # every size class is represented
    forms = {type(json.loads(b)["prompt"]).__name__ + ("" if not isinstance(json.loads(b)["prompt"], list) or not json.loads(b)["prompt"]
             else type(json.loads(b)["prompt"][0]).__name__) for b in bodies}
    assert {"str", "liststr", "listint", "listlist"} <= forms, forms
    kinds = b"".join(bodies)
    for needle in (b'"suffix"', b'"guided_json"', b'"logit_bias"', b'"stream_options"', b'"stream":true', b'"stop"', b'"seed"', b'"top_k"', b"\n  "):
        assert needle in kinds or needle.replace(b":", b": ") in kinds, needle


def test_edge_corpus_generator():
    bodies = edge_corpus()
    verdicts = [Q.parse_body(b)[0] for b in bodies]
    assert {Q.OK, Q.FAIL, Q.OUT} <= set(verdicts)
    assert Q.parse_body(_with("max_tokens", b"9223372036854775807"))[0] == Q.OK
    assert Q.parse_body(_with("max_tokens", b"9223372036854775808"))[0] == Q.FAIL
    for b in class_bound_bodies():
        assert Q.parse_body(b)[0] == Q.OK
    assert sorted({len(b) for b in class_bound_bodies()})[-1] == MAX_BODY + 1


def test_capacity_bodies():
    for ktok, classes in ((E.KTOK, E.CLASSES), ({2048: E.SMALL_KTOK, 5120: E.SMALL_KTOK}, (2048, 5120))):
        for c, k, fit, over in capacity_cases(ktok, classes):
            assert len(fit) == len(over) and E.PREV[c] < len(fit) <= c, (c, len(fit))
            assert E.count_tokens(fit) <= ktok[c] < E.count_tokens(over), (c, k)
            assert E.count_tokens(over) - E.count_tokens(fit) == 2
            assert Q.parse_body(fit)[0] == Q.OK and Q.parse_body(over)[0] == Q.OK
            assert json.loads(fit)["prompt"][:2] == [10000, 17919] and len(json.loads(over)["prompt"]) == k + 1


def test_mutation_seeds():
    seeds = mutation_seeds()
    assert len(seeds) >= MUTATION_SEEDS and all(Q.parse_body(s)[0] == Q.OK or s in [u["wrapped"].encode() for u in GOLD["unions"]] for s in seeds)
    assert sum(1 for s in seeds for _ in E.mutants(s)) > 5000
