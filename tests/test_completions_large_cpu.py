"""Corpora of /v1/completions requests for aigw_completions_translate_large_* (test_completions_large_gpu.py feeds them through the
GPU): seeded requests of 64 KiB to 8 MiB (fill-in-the-middle code, string batches, token-id prompts and token-id batches), bodies
with a flat id array's '[', an element, a comma or its ']' at every thread, warp and tile boundary of the scan and of the flat-array
stage's token partition, bodies at the limits, and probes that break a large flat prompt on those boundaries.  Here: their shape,
that they are reproducible, and the oracle's verdicts."""
import functools
import hashlib
import json
import random

import _completions_request_oracle as Q
import test_completions_request_cpu as G
import test_translate_edges_cpu as E

TILE, WARP, THREAD = 8192, 1024, 32   # the scan: bytes per round, per warp, per thread
FLAT_PER, FLAT_TILE = 8, 2048        # the flat-array stage: tokens per thread, per round
KINDS = ("fim", "string_batch", "tokens", "token_batch")


# ================================================================ realistic large requests
def _source(r, n):
    """about n characters of source text"""
    out = []
    size = 0
    while size < n:
        out.append(r.choice(G.CODE))
        size += len(out[-1])
    return "".join(out)


def _ids(r, n):
    return [r.randint(0, 200_000) for _ in range(n)]


def large_request(seed, target, kind):
    """a request of about `target` bytes: the sampling members and vLLM extras of test_completions_request_cpu's generator around a
    large prompt of the given kind"""
    r = random.Random(seed)
    ascii_, indent, compact = r.random() < 0.4, 2 if r.random() < 0.25 else None, r.random() < 0.5
    req = json.loads(G.realistic_request(seed))
    req.pop("suffix", None)
    if kind == "fim":
        req["prompt"] = _source(r, target * 3 // 4)
        req["suffix"] = _source(r, target // 4)
    elif kind == "string_batch":
        n = r.randint(2, 12)
        req["prompt"] = [_source(r, target // n) for _ in range(n)]
    elif kind == "tokens":
        req["prompt"] = _ids(r, target // 8)
    else:
        n = r.randint(2, 6)
        req["prompt"] = [_ids(r, target // (8 * n)) for _ in range(n)]
    return json.dumps(req, ensure_ascii=ascii_, indent=indent, separators=(",", ":") if compact else None).encode()


@functools.lru_cache(maxsize=None)
def realistic_corpus(n=18, lo=(64 << 10) + 8192, hi=8 << 20):
    """sizes spread log-uniformly between 64 KiB and 8 MiB, the four kinds in turn; a pretty-printed id prompt is about 1.7 times
    its compact size, so a body above 8 MiB is made again from a smaller target"""
    r = random.Random(2025)
    out = []
    for i in range(n):
        target = max(lo, min(hi, int(2 ** r.uniform(16, 23))))
        b = large_request(700 + i, target, KINDS[i % len(KINDS)])
        if len(b) > hi:
            b = large_request(700 + i, target * hi // len(b) * 15 // 16, KINDS[i % len(KINDS)])
        out.append(b)
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
IDS = [b"%d" % (100000 + (j * 7919) % 100000) for j in range(64)]   # six digits each: element j of an array starts at 1 + 7j
EDGES = (THREAD, WARP, TILE, 2 * TILE, 3 * TILE)
FEATURES = ("open", "elem", "comma", "close")


def _feature_offset(feature, arr):
    return {"open": 0, "elem": 1 + 20 * 7, "comma": 1 + 20 * 7 + 6, "close": len(arr) - 1}[feature]


def byte_placed(feature, at):
    """a body whose 40-id prompt has its '[', its 21st id, the comma after it or its ']' at byte `at`; a suffix string in front"""
    arr = b"[" + b",".join(IDS[:40]) + b"]"
    off = _feature_offset(feature, arr)
    head, mid = b'{"model":"m","suffix":"', b'","prompt":'
    pad = at - off - len(head) - len(mid)
    if pad < 0:
        return None
    body = head + b"a" * pad + mid + arr + b',"max_tokens":16}'
    assert body[at] == arr[off]
    return body


def _shift(s):
    """members in front of the prompt that add exactly s scan tokens (s >= 7): an unknown flat array of 2k + 5 tokens, and
    `"y":0,` (5) to make the count even"""
    tail = b""
    if s % 2 == 0:
        tail, s = b'"y":0,', s - 5
    k = (s - 5) // 2
    assert k >= 1
    return b'"x":[' + b",".join([b"0"] * k) + b"]," + tail


def token_placed(feature, t):
    """a body whose prompt has its '[', its 21st id, the comma after it or its ']' at scan token t (30 ids for ']'), with trailing
    white space that keeps it within the large call's len / 2 + 1024 tokens"""
    n = 30 if feature == "close" else 40
    a = t - {"open": 0, "elem": 41, "comma": 42, "close": 2 * n}[feature]   # the prompt's '[' token
    head = b'{"model":"m",' + _shift(a - 10) + b'"prompt":'
    arr = b"[" + b",".join(IDS[:n]) + b"]"
    body = head + arr + b"}"
    at = len(head) + _feature_offset(feature, arr)
    assert E.count_tokens(body[:at]) == t and body[at] == arr[_feature_offset(feature, arr)], (feature, t)
    return body + b" " * max(0, 2 * (E.count_tokens(body) - 1024) + 64 - len(body))


T_EDGES = (16 * FLAT_PER, FLAT_TILE, 2 * FLAT_TILE)


@functools.lru_cache(maxsize=None)
def boundary_bodies():
    """each feature within +-40 bytes of every thread, warp and tile boundary of the scan, within +-10 tokens of the flat stage's
    round boundaries (crossing per-thread boundaries on the way), and bodies of 65535-65537 bytes"""
    out = []
    for feature in FEATURES:
        for edge in EDGES:
            for delta in range(-40, 41, 4):
                b = byte_placed(feature, edge + delta)
                if b is not None:
                    out.append(b)
        for edge in T_EDGES:
            for delta in range(-10, 11):
                out.append(token_placed(feature, edge + delta))
    out += [G.token_prompt_body(2000, n) for n in (65535, 65536, 65537, 65536 + TILE)]
    return tuple(out)


def deep(d):
    """nesting depth d, the innermost array flat, under a member the request ignores"""
    v = "[1,2,3]"
    for _ in range(d - 2):
        v = "[" + v + "]"
    return ('{"model":"m","prompt":[1,2],"x":' + v + "}").encode()


def near_16mib():
    """16 MiB - 1 bytes: a 600 000-id prompt (about 4.2 MB) after a fill-in-the-middle suffix"""
    ids = b",".join(b"%d" % (100000 + (j * 7919) % 100000) for j in range(600_000))
    head, mid = b'{"model":"m","stream":true,"suffix":"', b'","prompt":[' + ids + b"]}"
    return head + b"s" * ((16 << 20) - 1 - len(head) - len(mid)) + mid


def token_edge(k, length):
    """a prompt of k one-byte ids, padded to `length`: 2k + 12 scan tokens"""
    s = b'{"model":"m","prompt":[' + b",".join([b"1"] * k) + b"]}"
    return s + b" " * (length - len(s))


TOKEN_K = 3000
TOKEN_LEN = 4 * TOKEN_K - 2024   # 2k + 12 tokens == length / 2 + 1024


# ================================================================ probes in a large flat prompt
# an element of a []int64 prompt replaced by the probe
ELEMENT_PROBES = {
    "letter": b"12a45", "double_comma": b"", "space": b"1 2", "nested": b"[2]", "string": b'"2"', "true": b"true", "null": b"null",
    "frac": b"1.5", "exp": b"1e2", "neg_zero": b"-0", "leading_zero": b"01", "max": b"9223372036854775807",
    "max+1": b"9223372036854775808", "max-1": b"9223372036854775806", "min": b"-9223372036854775808", "min-1": b"-9223372036854775809",
    "min+1": b"-9223372036854775807", "digits20": b"12345678901234567890", "digits19": b"1000000000000000000", "zero": b"0",
}
# (token of the probed element, byte of the probe's first byte): the flat stage's round and thread boundaries, the scan's tiles,
# warps and threads, and one past the translate pass's 64 KiB ceiling
PLACEMENTS = ((2047, 2 * TILE), (2049, 3 * TILE + WARP), (4095, 4 * TILE + THREAD), (4097, 9 * TILE), (6143, 9 * TILE - 1))
HEAD = b'{"model":"m","suffix":"'   # then a pad string, then '","prompt":[', whose '[' is token 16


def _placed(at, before, after):
    """HEAD, a pad string, `before`, `after`: the first byte of `after` at byte `at`"""
    pad = at - len(HEAD) - len(before)
    assert pad >= 0, (at, len(before))
    body = HEAD + b"p" * pad + before + after
    assert body[at:at + len(after[:1])] == after[:1]
    return body


def _ids_text(n):
    return [b"%d" % (100000 + (j * 7919) % 100000) for j in range(n)]


def element_probe(probe, t, at):
    """a flat prompt whose element at scan token t (odd: the '[' is token 16) is `probe`, its first byte at byte `at`"""
    i = (t - 17) // 2
    ids = _ids_text(i + 300)
    body = _placed(at, b'","prompt":[' + b"".join(x + b"," for x in ids[:i]), probe + b"," + b",".join(ids[i + 1:]) + b'],"max_tokens":64}')
    assert not probe or E.count_tokens(body[:at]) == t, (probe, t, at)
    return body


def structure_probes(t, at):
    """probes of the array's own structure, of batches and of the other members' flat arrays, their first byte at `at`: name → body"""
    ids = _ids_text((t - 17) // 2)
    pre = b",".join(ids)
    rest = b"," + b",".join(_ids_text(300)) + b"]"
    mid = b'","prompt":['
    return {
        # [1,] and [,1]: a trailing comma ends the prompt; a leading one starts an inner array of a batch
        "trailing_comma": _placed(at, mid + pre, b",]}"),
        "leading_comma": _placed(at, mid + b"[" + pre + b"],", b"[,1,2]]}"),
        "inner_empty": _placed(at, mid + b"[" + pre + b"],", b"[]]}"),
        "inner_null": _placed(at, mid + b"[" + pre + b"],", b"null]}"),
        "inner_string": _placed(at, mid + b"[" + pre + b"],[1,", b'"x",2]]}'),
        "inner_nested": _placed(at, mid + b"[" + pre + b"],[1,", b"[2],3]]}"),
        "inner_float": _placed(at, mid + b"[" + pre + b"],[1,", b"2.0,3]]}"),
        "batch_scalar": _placed(at, mid + b"[" + pre + b"],", b"3]}"),
        "first_null": _placed(at, mid, b"null," + pre + rest + b"}"),
        "empty_in_batch": _placed(at, mid, b"[],[" + pre + b"]]}"),
        # [] and [[]]: nothing to check; the pad carries the size
        "empty": _placed(at, mid, b"]}"),
        "empty_inner": _placed(at, mid, b"[]]}"),
        # flat number arrays in stop (float64: an exponent or more than 308 integer digits declines) and in an unknown member
        "stop_exp": _placed(at, b'","stop":[' + pre + b",", b"1e5,7]}"),
        "stop_309": _placed(at, b'","stop":[' + pre + b",", b"1" * 309 + b",7]}"),
        "stop_308": _placed(at, b'","stop":[' + pre + b",", b"9" * 308 + b",7]}"),
        "stop_frac": _placed(at, b'","stop":[' + pre + b",", b"-2.5,7]}"),
        "unknown_exp": _placed(at, b'","x_ids":[' + pre + b",", b'1e400,7],"prompt":[1,2]}'),
        "unknown_true": _placed(at, b'","x_ids":[' + pre + b",", b'true,7],"prompt":[1,2]}'),
    }


@functools.lru_cache(maxsize=None)
def probe_corpus():
    """(label, body): every element probe and structure probe at every placement"""
    out = []
    for t, at in PLACEMENTS:
        for name, probe in ELEMENT_PROBES.items():
            out.append(("%s t%d b%d" % (name, t, at), element_probe(probe, t, at)))
        for name, body in structure_probes(t, at).items():
            out.append(("%s t%d b%d" % (name, t, at), body))
    return tuple(out)


# the oracle's verdict of each probe (the same at every placement)
PROBE_VERDICTS = {
    "letter": Q.FAIL, "double_comma": Q.FAIL, "space": Q.FAIL, "nested": Q.FAIL, "string": Q.FAIL, "true": Q.FAIL, "null": Q.OK,
    "frac": Q.FAIL, "exp": Q.FAIL, "neg_zero": Q.OK, "leading_zero": Q.FAIL, "max": Q.OK, "max+1": Q.FAIL, "max-1": Q.OK, "min": Q.OK,
    "min-1": Q.FAIL, "min+1": Q.OK, "digits20": Q.FAIL, "digits19": Q.OK, "zero": Q.OK,
    "trailing_comma": Q.FAIL, "leading_comma": Q.FAIL, "inner_empty": Q.OK, "inner_null": Q.OK, "inner_string": Q.FAIL,
    "inner_nested": Q.FAIL, "inner_float": Q.FAIL, "batch_scalar": Q.FAIL, "first_null": Q.FAIL, "empty_in_batch": Q.OK, "empty": Q.OK,
    "empty_inner": Q.OK, "stop_exp": Q.OUT, "stop_309": Q.OUT, "stop_308": Q.OK, "stop_frac": Q.OK, "unknown_exp": Q.OK,
    "unknown_true": Q.OK,
}


def digest(bodies):
    h = hashlib.sha256()
    for b in bodies:
        h.update(len(b).to_bytes(8, "little")); h.update(b)
    return h.hexdigest()


# ================================================================ tests
DIGESTS = {
    "realistic": "9e386b2e3b82ea1a49282322c278289659c49d5a2c11f281ea3555c50e4aa3e7",
    "boundary": "bc1483cfa79a56d19ec656fae931e971ef98077f1f05679d444426e1197683c6",
    "probe": "bab80d6cba1abcbd6ccc89efa46cc4290c556365fd1f8690d8714b601728b3c0",
}


def test_corpus_shape_and_reproducible():
    c = realistic_corpus()
    # pinned: a change to the generator changes what the GPU tests compare, and shows here
    assert digest(c) == DIGESTS["realistic"]
    assert digest(boundary_bodies()) == DIGESTS["boundary"]
    assert digest(b for _, b in probe_corpus()) == DIGESTS["probe"]
    sizes = [len(b) for b in c]
    assert min(sizes) >= 64 << 10 and max(sizes) <= 9 << 20 and max(sizes) >= 2 << 20, sizes
    assert 20 << 20 <= sum(sizes) <= 45 << 20, sum(sizes)
    forms = set()
    for b in c:
        p = json.loads(b)["prompt"]
        forms.add(type(p).__name__ + (type(p[0]).__name__ if isinstance(p, list) else ""))
        if isinstance(p, list) and isinstance(p[0], int):
            assert max(p) > 150_000 and len(p) > 6000
    assert forms == {"str", "liststr", "listint", "listlist"}, forms
    assert any(b'"suffix"' in b for b in c)
    assert any(max(b) >= 0x80 for b in c) and any(max(b) < 0x80 for b in c)    # ensure_ascii off and on
    assert any(b"\n  " in b for b in c) and any(b"\n" not in b for b in c)      # pretty-printed and compact
    extras = b"".join(c)
    for needle in (b'"max_tokens"', b'"stream"', b'"temperature"'):
        assert needle in extras, needle
    assert any(k in extras for k in (b'"top_k"', b'"min_p"', b'"guided_json"', b'"stop_token_ids"', b'"repetition_penalty"'))


def test_oracle_accepts_realistic():
    for b in realistic_corpus():
        v, model, stream = verdict(b)
        j = json.loads(b)
        assert v == Q.OK and model == j["model"].encode() and stream == bool(j.get("stream")), len(b)


def test_boundary_shapes():
    bb = boundary_bodies()
    assert len(bb) > 500
    for b in bb:
        assert verdict(b)[0] == Q.OK, b[:120]
    assert sorted(len(b) for b in bb)[-4:] == [65535, 65536, 65537, 65536 + TILE]
    # the flat stage's round edges are crossed by every feature, and so are per-thread edges (multiples of 8) on the way
    for feature in FEATURES:
        for t in (FLAT_TILE - 1, FLAT_TILE, 2 * FLAT_TILE + 1):
            assert token_placed(feature, t) in bb


def test_limit_shapes():
    assert verdict(deep(48))[0] == Q.OK and verdict(deep(49))[0] == Q.OUT and json.loads(deep(49))
    big = near_16mib()
    assert len(big) == (16 << 20) - 1 and len(json.loads(big)["prompt"]) == 600_000
    at, over = token_edge(TOKEN_K, TOKEN_LEN), token_edge(TOKEN_K + 1, TOKEN_LEN)
    assert len(at) == len(over) == TOKEN_LEN
    assert E.count_tokens(at) == TOKEN_LEN // 2 + 1024 == E.count_tokens(over) - 2
    assert verdict(at)[0] == verdict(over)[0] == Q.OK


def test_probe_corpus():
    """each probe sits on its boundary (asserted as it is built) and gets the oracle verdict the table gives it"""
    pc = probe_corpus()
    assert len(pc) == len(PLACEMENTS) * len(PROBE_VERDICTS)
    for label, b in pc:
        assert verdict(b)[0] == PROBE_VERDICTS[label.split(" ")[0]], label
