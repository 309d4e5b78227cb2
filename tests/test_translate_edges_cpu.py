"""Generators for the translate pass's layout-edge tests (test_translate_edges_gpu.py), and their self-checks (no GPU).

The chat translate kernels work in fixed units: size classes of 2048 … 65536 input bytes, a token capacity kTok per class,
32-byte lane blocks, 1 KiB index rounds, 16-byte emit chunks in tiles of 256.  The helpers here build bodies that sit exactly
on those numbers: bodies of an exact byte length, bodies with an exact token count, and a feature slid across a boundary.
`count_tokens` restates the index stage's token definition (chat_stage.cuh index_doc) in plain Python."""
import json

import pytest

import _oracle as O

CLASSES = (2048, 5120, 9216, 17408, 33792, 65536)
PREV = dict(zip(CLASSES, (0,) + CLASSES[:-1]))   # class c holds bodies of (PREV[c], c] bytes
SMALL_MAX = 5120                                   # the fused small-batch kernel takes bodies up to this length
REASON_TOO_LARGE, REASON_TOKENS, REASON_DEPTH = 1, 5, 16
CAPACITY_REASONS = (5, 6, 7)                       # tokens, ops, scratch


def ktok(maxd):
    """Cls<MAXD>::kTok (chat_kernel.cuh): about one token per 8 input bytes, at least 512, rounded up to 64."""
    return 512 if maxd // 8 < 512 else (maxd // 8 + 63) // 64 * 64


KTOK = {c: ktok(c) for c in CLASSES}
SMALL_KTOK = KTOK[SMALL_MAX]


def class_of(n):
    return next((c for c in CLASSES if n <= c), CLASSES[-1])


# ---------------------------------------------------------------- token count (restates index_doc)
_WS = frozenset(b" \t\n\r")
_OPS = frozenset(b"{}[]:,")


def count_tokens(body: bytes) -> int:
    """One token per unescaped quote, per structural byte {}[]:, outside strings, and per start of a run of scalar bytes
    (neither structural nor whitespace) outside strings.  A byte is escaped when an odd run of backslashes precedes it,
    whether or not it is inside a string, as the index stage computes it."""
    n = 0
    in_str = False
    run = 0          # backslashes immediately before the current byte
    prev_scalar = False
    for c in body:
        escaped = run & 1
        run = run + 1 if c == 0x5C else 0
        if c == 0x22 and not escaped:
            n += 1
            in_str = not in_str
            prev_scalar = False
        elif in_str:
            prev_scalar = False
        elif c in _OPS:
            n += 1
            prev_scalar = False
        elif c in _WS:
            prev_scalar = False
        else:
            n += not prev_scalar
            prev_scalar = True
    return n


# ---------------------------------------------------------------- bodies of an exact length
FILL = b"lorem ipsum dolor sit amet, consectetur adipiscing elit; "
MARK = b"@@"

TEMPLATES = {
    "aws-bedrock": b'{"model":"m","messages":[{"role":"system","content":"be brief"},{"role":"user","content":"@@"}],"max_tokens":7}',
    "openai": b'{"model":"m","messages":[{"role":"system","content":"be brief"},{"role":"user","content":"@@"}],"max_tokens":7}',
    "gcp-vertexai": b'{"model":"gemini-2.5-flash","messages":[{"role":"user","content":"@@"}],"max_tokens":7}',
    "msg-openai": b'{"model":"claude-3","max_tokens":16,"messages":[{"role":"user","content":"@@"}]}',
}


def fill(k: int, start: int = 0) -> bytes:
    reps = (start + k) // len(FILL) + 2
    return (FILL * reps)[start:start + k]


def pad_to(template: bytes, n: int) -> bytes:
    """template with its one @@ replaced by filler text, so that the body is exactly n bytes long"""
    k = n - (len(template) - len(MARK))
    assert k >= 0, (n, len(template))
    return template.replace(MARK, fill(k), 1)


def oracle(schema, body: bytes):
    """the reference translation of `body` for a GPU schema name"""
    if schema == "msg-openai":
        return O.messages_translate("openai", body, api_version="v1")
    return O.chat_translate(schema, body, prefix="" if "anthropic" in schema else "v1")


def out_len(schema, body):
    """path + body bytes of the reference's record (what the emit stage writes), or None when the reference does not translate"""
    o = oracle(schema, body)
    if o.status != O.OK:
        return None
    return len(o.path.encode()) + (len(o.body) if o.body_kind == O.BYTES else 0)


def size_class_bodies(schema):
    """A1: bodies of exactly c-16, c-1, c, c+1 bytes for every class bound c (no c+1 above the largest class)"""
    t = TEMPLATES[schema]
    out = []
    for c in CLASSES:
        for n in (c - 16, c - 1, c, c + 1):
            if n <= CLASSES[-1]:
                out.append(pad_to(t, n))
    return out


def too_large_body(schema="aws-bedrock"):
    return pad_to(TEMPLATES[schema], CLASSES[-1] + 1)


def aligned_output_bodies(schema="aws-bedrock"):
    """A1: rewritten records that end exactly on a 16-byte boundary in every class, and records of 4095 … 4113 bytes around the
    emit kernel's 256-chunk tile; lengths found by scanning the filler length against the reference."""
    t = TEMPLATES[schema]
    out = []
    for c in CLASSES:
        for n in range(c - 40, c + 1):
            b = pad_to(t, n)
            if out_len(schema, b) % 16 == 0:
                out.append(b)
                break
    base = out_len(schema, pad_to(t, 200)) - 200   # the record grows byte for byte with the plain filler
    for want in (4080, 4095, 4096, 4097, 4112, 4113, 8192):
        b = pad_to(t, want - base)
        assert out_len(schema, b) == want
        out.append(b)
    return out


# ---------------------------------------------------------------- bodies of an exact token count
STOP_TEMPLATE = b'{"model":"m","messages":[{"role":"user","content":"@@"}]%s,"stop":[%s]}'
EXTRAS = (b"", b',"n":1', b',"temperature":1,"n":1')   # +0, +5, +10 tokens: with the stop array's 3k-1 every residue is reachable


def token_body(tokens: int, length: int) -> bytes:
    """an OpenAI-schema body with exactly `tokens` tokens and `length` bytes: a stop array of k one-letter strings sets the
    count, the content string (two tokens whatever its length) sets the length"""
    for extra in EXTRAS:
        base = count_tokens(STOP_TEMPLATE % (extra, b""))
        k, r = divmod(tokens - base + 1, 3)
        if r == 0 and k >= 1:
            t = STOP_TEMPLATE % (extra, b",".join([b'"a"'] * k))
            b = pad_to(t, length)
            assert count_tokens(b) == tokens and len(b) == length
            return b
    raise AssertionError((tokens, length))


def token_cases():
    """A2: (class, tokens, body).  Pipeline: kTok and kTok+1 inside each class's length range.  Fused kernel (bodies ≤ 5120): its own
    capacity of 640 and 641, once in the 5120 class and once in the 2048 class, where the pipeline's capacity is 512."""
    out = []
    for c in CLASSES:
        n = max(PREV[c] + 1, min(c, 5 * KTOK[c] + 400))   # inside (PREV[c], c] with room for the stop array
        for t in (KTOK[c] - 1, KTOK[c], KTOK[c] + 1):
            out.append((c, t, token_body(t, n)))
    for t in (SMALL_KTOK, SMALL_KTOK + 1):
        out.append((2048, t, token_body(t, 2048)))
    return out


# ---------------------------------------------------------------- features slid across lane and round boundaries
STRADDLE_HEAD = b'{"model":"m","messages":[{"role":"user","content":"'
SURROGATE = b"\\ud83d\\ude00"
STRING_FEATURES = {   # inside the user content string; the offset is that of the feature's first byte
    "esc_quote": b'\\"', "esc_bslash": b"\\\\", "esc_slash": b"\\/", "esc_b": b"\\b", "u_e9": b"\\u00e9", "surrogate": SURROGATE,
    "utf8_4": "\U0001F600".encode(), "bs3_quote": b'\\\\\\"', "bs5_quote": b'\\\\\\\\\\"', "bs1_quote": b'\\"',
}


def straddle_body(feature: str, at: int, length: int) -> bytes:
    """a body of `length` bytes whose feature starts at byte offset `at` (a byte of it may straddle a 32-byte block or a 1 KiB round)"""
    if feature in STRING_FEATURES:
        f = STRING_FEATURES[feature]
        pre = at - len(STRADDLE_HEAD)
        tail = b'"}],"max_tokens":7}'
        post = length - at - len(f) - len(tail)
        return STRADDLE_HEAD + fill(pre) + f + fill(post, pre) + tail
    if feature in ("bs2_close", "bs4_close"):   # an even backslash run, then the quote that closes the string: the quote is at `at`
        k = 2 if feature == "bs2_close" else 4
        pre = at - k - len(STRADDLE_HEAD)
        mid = b'"}],"max_tokens":7,"user":"'
        post = length - at - len(mid) - 2
        return STRADDLE_HEAD + fill(pre) + b"\\" * k + mid + fill(post) + b'"}'
    if feature == "number":   # "max_tokens":1234567 with the number's first digit at `at`
        key = b'"}],"max_tokens":'
        pre = at - len(key) - len(STRADDLE_HEAD)
        rest = b',"user":"'
        post = length - at - 7 - len(rest) - 2
        return STRADDLE_HEAD + fill(pre) + key + b"1234567" + rest + fill(post) + b'"}'
    if feature == "esc_key":   # the model key spelled with an escape, its opening quote at `at`
        head = b'{"messages":[{"role":"user","content":"'
        key = b'"}],"\\u006dodel":"m","user":"'
        pre = at - len(head) - 4
        post = length - at - (len(key) - 4) - 2
        return head + fill(pre) + key + fill(post) + b'"}'
    raise KeyError(feature)


FEATURES = tuple(STRING_FEATURES) + ("bs2_close", "bs4_close", "number", "esc_key")


def round_boundaries(c):
    """the first, a middle and the last 1 KiB round boundary of class c"""
    last = (c - 1) // 1024 * 1024
    return sorted({1024, (last // 2048) * 1024 or 1024, last})


def straddle_cases(window=40):
    """A3: (class, boundary, feature, body) for every offset in ±window around a lane boundary and the round boundaries"""
    out = []
    for c in CLASSES:
        bounds = ([512] if c == CLASSES[0] else []) + round_boundaries(c)
        for bnd in bounds:
            length = max(PREV[c] + 1, min(c, bnd + 200))
            for f in FEATURES:
                for at in range(bnd - window, bnd + window + 1):
                    out.append((c, bnd, f, straddle_body(f, at, length)))
    return out


def long_string_cases():
    """A3: strings longer than 2 KiB (they span several words of the per-round escape mask) with a re-spelled escape \\/ only in the
    string's first 32-byte block, only in its last block, or in neither; the string start slides so that the last block takes
    every position inside its mask word"""
    out = []
    for where in ("first", "last", "none"):
        for shift in range(0, 64, 3):
            n_str = 2100 + 37 * shift
            s = bytearray(fill(n_str))
            if where == "first":
                s[0:2] = b"\\/"
            elif where == "last":
                s[-2:] = b"\\/"
            body = b'{"model":"m","messages":[{"role":"system","content":"' + fill(shift) + b'"},{"role":"user","content":"' + bytes(s) + b'"}],"max_tokens":7}'
            out.append((where, shift, body))
    return out


# ---------------------------------------------------------------- nesting depth
def depth_body(kind: str, k: int) -> bytes:
    """a valid body with k nested arrays inside a member the translator walks into"""
    inner = b"[" * k + b"1" + b"]" * k
    if kind == "passthrough":   # an unknown top-level field: validated, forwarded untouched
        return b'{"model":"m","messages":[{"role":"user","content":"hi"}],"x_nested":' + inner + b"}"
    if kind == "tool_args":     # a tool call's arguments object: parsed and re-emitted as the toolUse input
        a = json.dumps({"a": json.loads(inner)}, separators=(",", ":"))
        return (b'{"model":"m","messages":[{"role":"user","content":"hi"},{"role":"assistant","tool_calls":[{"id":"c1","type":"function","function":{"name":"f","arguments":'
                + json.dumps(a).encode() + b"}}]}]}")
    if kind == "gemini_params":   # a tool's parameters schema: nested array items
        p = b'{"type":"object","properties":{"a":' + b'{"type":"array","items":' * k + b'{"type":"string"}' + b"}" * k + b"}}"
        return (b'{"model":"gemini-2.5-flash","messages":[{"role":"user","content":"hi"}],"tools":[{"type":"function","function":{"name":"f","parameters":'
                + p + b"}}]}")
    raise KeyError(kind)


DEPTH_SCHEMA = {"passthrough": "openai", "tool_args": "aws-bedrock", "gemini_params": "gcp-vertexai"}


# ---------------------------------------------------------------- structural mutation corpus
MUTATION_BYTES = b'{}[]:,"\\ '


def mutation_seeds():
    """(schema, body): about 30 small valid bodies of different shapes"""
    S = []
    for schema in ("aws-bedrock", "openai", "gcp-vertexai"):
        S += [
            (schema, b'{"model":"m","messages":[{"role":"user","content":"hi"}]}'),
            (schema, b'{"model":"m","messages":[{"role":"system","content":"s"},{"role":"user","content":[{"type":"text","text":"a\\"b"}]}],"max_tokens":5}'),
            (schema, b'{"model":"m","messages":[{"role":"user","content":"x"}],"temperature":0.5,"top_p":1,"stop":["a","b"],"stream":true}'),
            (schema, b'{ "model" : "m" , "messages" : [ { "role" : "user" , "content" : "t\\u00e9\\n" } ] , "max_tokens" : 10 }'),
            (schema, b'{"messages":[{"role":"assistant","content":null,"tool_calls":[{"id":"c","type":"function","function":{"name":"f","arguments":"{\\"a\\":[1,{\\"b\\":null}]}"}}]},{"role":"tool","tool_call_id":"c","content":"ok"}],"model":"m"}'),
            (schema, b'{"model":"m","messages":[{"role":"user","content":"q"}],"tools":[{"type":"function","function":{"name":"f","description":"d","parameters":{"type":"object","properties":{"x":{"type":"string"}},"required":["x"]}}}],"tool_choice":"auto"}'),
            (schema, b'{"model":"m","messages":[{"role":"developer","content":[{"type":"text","text":"p"},{"type":"text","text":"q"}]},{"role":"user","content":"r","name":"bob"}],"n":1,"seed":42}'),
            (schema, b'{"model":"m","messages":[],"stream":true,"stream_options":{"include_usage":true},"user":"u"}'),
            (schema, b'{"model":"m","messages":[{"role":"user","content":"\\\\ end"}],"max_completion_tokens":1024,"metadata":{"k":[true,false,null]}}'),
            (schema, b'{"model":"m","messages":[{"role":"assistant","content":"a"},{"role":"user","content":"b"}],"stop":"END","presence_penalty":-0.25}'),
        ]
    # Gemini: assistant tool calls and tool_choice are left to the stock path by both sides; a tool schema and nested parts instead
    gem = [(b"gcp-vertexai", b'{"model":"m","messages":[{"role":"user","content":"q"}],"tools":[{"type":"function","function":{"name":"f","parameters":{"type":"object","properties":{"n":{"type":"string","enum":["a","b"]}}}}}]}'),
           (b"gcp-vertexai", b'{"model":"m","messages":[{"role":"system","content":[{"type":"text","text":"s"}]},{"role":"user","content":[{"type":"text","text":"t"}]}],"top_p":0.5}')]
    S = [x for x in S if not (x[0] == "gcp-vertexai" and (b"tool_calls" in x[1] or b"tool_choice" in x[1]))] + [(s.decode(), b) for s, b in gem]
    return S


def mutants(body: bytes):
    """every one-byte mutation of body: delete, duplicate, or replace with one of {}[]:," \\ and space (identical results dropped)"""
    seen = set()
    for i in range(len(body)):
        cands = [body[:i] + body[i + 1:], body[:i + 1] + body[i:i + 1] + body[i + 1:]]
        cands += [body[:i] + bytes([c]) + body[i + 1:] for c in MUTATION_BYTES if c != body[i]]
        for m in cands:
            if m not in seen and m != body:
                seen.add(m)
                yield m


# ================================================================ self-checks
def test_token_counter_known_answers():
    cases = [(b"{}", 2), (b'{"a":1}', 6), (b"[1, 22 ,true]", 7), (b'{"a\\"b":"c\\\\"}', 7), (b'"x" "y"', 4), (b"12 34", 2), (b"1,2", 3),
             (b'"a\\\\\\"b"', 2), (b'{"k":-1.5e3,"v":[null]}', 13), (b"  \t\n{ }\r\n", 2), (b'"{[:,]}"', 2), (b"", 0), (b"tru e", 2),
             (b'\\"x', 1)]   # outside strings an escaped quote is a scalar byte: `\"x` is one scalar run, and so is nothing else
    for b, want in cases:
        assert count_tokens(b) == want, (b, count_tokens(b), want)


def test_ktok_table():
    assert KTOK == {2048: 512, 5120: 640, 9216: 1152, 17408: 2176, 33792: 4224, 65536: 8192}


@pytest.mark.parametrize("schema", list(TEMPLATES))
def test_exact_length_helper(schema):
    bodies = size_class_bodies(schema)
    want = [n for c in CLASSES for n in (c - 16, c - 1, c, c + 1) if n <= CLASSES[-1]]
    assert [len(b) for b in bodies] == want
    for b in bodies[::5]:
        json.loads(b)
        assert oracle(schema, b).status == O.OK, schema
    assert len(too_large_body(schema)) == 65537


def test_aligned_output_bodies():
    bodies = aligned_output_bodies()
    lens = [out_len("aws-bedrock", b) for b in bodies]
    assert all(n % 16 == 0 for n in lens[:len(CLASSES)])
    assert lens[len(CLASSES):] == [4080, 4095, 4096, 4097, 4112, 4113, 8192]
    assert [class_of(len(b)) for b in bodies[:len(CLASSES)]] == list(CLASSES)


def test_token_bodies_hit_capacity():
    cases = token_cases()
    for c, t, b in cases:
        assert count_tokens(b) == t and PREV[c] < len(b) <= c, (c, t, len(b))
        assert oracle("openai", b).status == O.OK
        json.loads(b)
    got = {(c, t) for c, t, _ in cases}
    for c in CLASSES:
        assert (c, KTOK[c]) in got and (c, KTOK[c] + 1) in got
    assert (2048, 640) in got and (2048, 641) in got and (5120, 640) in got and (5120, 641) in got


def test_straddle_bodies():
    cases = straddle_cases(window=3)
    for c, bnd, f, b in cases:
        assert PREV[c] < len(b) <= c, (c, bnd, f, len(b))
        json.loads(b)
        o = oracle("aws-bedrock", b)
        assert o.status == O.OK, (f, bnd, o.err)
    # the feature is where it is claimed to be
    b = straddle_body("esc_slash", 1020, 1400)
    assert b[1020:1022] == b"\\/"
    b = straddle_body("bs4_close", 1030, 1400)
    assert b[1026:1031] == b'\\\\\\\\"'
    b = straddle_body("number", 1000, 1400)
    assert b[1000:1007] == b"1234567"
    b = straddle_body("esc_key", 1000, 1400)
    assert b[1000:1012] == b'"\\u006dodel"'
    assert {k for k in json.loads(b)} == {"messages", "model", "user"}
    for f in FEATURES:
        assert len(straddle_body(f, 2000, 2100)) == 2100


def test_long_string_bodies():
    for where, shift, b in long_string_cases():
        s = json.loads(b)["messages"][1]["content"]
        assert len(s) > 2048
        assert ("/" in s[:2]) == (where == "first") and ("/" in s[-2:]) == (where == "last")
        assert oracle("aws-bedrock", b).status == O.OK


@pytest.mark.parametrize("kind", list(DEPTH_SCHEMA))
def test_depth_bodies(kind):
    for k in (1, 20, 47, 60):
        b = depth_body(kind, k)
        json.loads(b)
        assert oracle(DEPTH_SCHEMA[kind], b).status == O.OK, (kind, k)


def test_mutation_corpus_shape():
    seeds = mutation_seeds()
    assert len(seeds) == 30
    for schema, b in seeds:
        json.loads(b)
        assert oracle(schema, b).status == O.OK, (schema, b)
    ms = list(mutants(b'{"a":1}'))
    assert len(ms) == len(set(ms)) and b'{"a":1}' not in ms
    assert b'{"a"1}' in ms and b'{{"a":1}' in ms and b'{"a":1]' in ms
    # a mutant is what it claims: one byte deleted, inserted or replaced
    for m in ms:
        assert abs(len(m) - 7) <= 1
