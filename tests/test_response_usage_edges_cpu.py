"""Edge corpora for the buffered response-usage kernels (sse_kernel.cu: response_usage_kernel for chat and embeddings,
completions_response_kernel for /v1/completions and /v1/responses, rerank_response_kernel) and a big-integer model of the CEL cost
VM (cel_kernel.cuh), with the self-checks that pin them on a machine without a GPU.  test_response_usage_edges_gpu.py runs them.

Expected record.  Every body gets one: (status, usage, model bytes), usage = (input, cached, cache_creation, output, total,
reasoning, mask) with 0 where the mask bit is clear.  It comes from
  * the verdict of `predict`, a typed walk of the kind's schema (the tuple tables below, in _responses_oracle's notation) that
    restates when the library declines: OUT → DECLINED, FAIL → INTERNAL ("failed to unmarshal body"), OK → decoded;
  * for OK: the C++ oracle's record for chat, embeddings and completions (oracle/oracle_capi.cpp), and the walk's own captures for
    /v1/responses and rerank, whose oracles are that walk (_responses_oracle, _rerank_oracle).
The self-checks below hold `predict` to the C++ oracle wherever it says OK or FAIL.

The decline rules restated (each is counted in RULES and must occur in the corpora):
  esc_key       an escaped member name inside a typed object (sonic may match it to a field after unescaping);
  dup_key       a repeated known member of a typed object, except the /v1/responses root's members from the 33rd on
                (presence_penalty, frequency_penalty, store), which the walk does not track (tjson.cuh: `EXT && f >= 32`);
  typed_depth   a non-empty typed object or array 13 deep (walk's MAXD = 12);
  skip_depth    an unknown member's value that opens a 65th level (skip_any's 64-level bitmask);
  esc_model     an escaped model string (chat, embeddings, completions, responses);
  big           completions only: a usage counter outside [0, 2^31) (the reference sets a counter only when it is >= 0);
  f64           rerank only: a float64 with an exponent or more than 308 integer digits, or a token count whose float64 lies outside
                (-1, 2^32), where Go's uint32 conversion is implementation-defined;
  union         /v1/responses only: an output item, tool or tool choice the schema knows but does not restate, an escaped tag, or a
                float32 with an exponent or more than 38 integer digits.

Nesting limit.  The reference pins sonic v1.15.1; its source is not available here, so its exact depth limit is unverified.  The C++
oracle's parser (oracle/ojson.hpp) accepts 512 levels and fails the 513th; sonic may differ there.  Past the kernel's own bounds
(12 typed levels, 64 skipped levels) the expected answer is DECLINED whatever the oracle says, never INTERNAL.
"""
import collections
import hashlib
import json
import os
import random

import numpy as np
import pytest

import _oracle as O
import _rerank_oracle as Q
import _responses_oracle as R
import test_cel_gpu as CG
import test_large_scan_defects_cpu as LD
import test_response_gpu as RG
import test_translate_edges_cpu as E

KINDS = ("chat", "embeddings", "completions", "responses", "rerank")
OK, INTERNAL, DECLINED = 0, 3, 4   # enum aigw_status
MUT_BYTES = E.MUTATION_BYTES + bytes(c for c in LD.MUT_BYTES if c not in E.MUTATION_BYTES)   # as test_walk_group_mutations_cpu
ZERO7 = (0,) * 7

# ---------------------------------------------------------------- schemas (sse_schema.cuh, in _responses_oracle's notation)
_FUNC = ("obj", {"arguments": "str", "name": "str"}, None)
_CACHE = ("obj", {"type": "str", "ttl": "str"}, None)
_TOOLCALL = ("obj", {"id": "str", "function": _FUNC, "type": "str", "cache_control": _CACHE}, None)
_URLCIT = ("obj", {"end_index": "int", "start_index": "int", "url": "str", "title": "str"}, None)
_ANNOT = ("obj", {"type": "str", "url_citation": _URLCIT}, None)
_AUDIO = ("obj", {"data": "str", "expires_at": "int", "id": "str", "transcript": "str"}, None)
_REASON_TEXT = ("obj", {"text": "str", "signature": "str"}, None)
_REASON_BLOCK = ("obj", {"reasoningText": _REASON_TEXT, "redactedContent": "b64"}, None)
_THINK = ("obj", {"type": "str", "thinking": "str", "signature": "str", "data": "str"}, None)
_TOPLP = ("obj", {"token": "str", "bytes": ("arr", "int"), "logprob": "float"}, None)
_TOKLP = ("obj", {"token": "str", "bytes": ("arr", "int"), "logprob": "float", "top_logprobs": ("arr", _TOPLP)}, None)
_LOGPROBS = ("obj", {"content": ("arr", _TOKLP), "refusal": ("arr", _TOKLP)}, None)
_MSG = ("obj", {"content": "str", "role": "str", "tool_calls": ("arr", _TOOLCALL), "annotations": ("arr", _ANNOT), "audio": _AUDIO,
                "reasoning_content": ("strobj", ("obj", {"reasoningContent": _REASON_BLOCK}, None)), "thinking_blocks": ("arr", _THINK),
                "safety_ratings": "any", "grounding_metadata": "any"}, None)
_CHOICE = ("obj", {"finish_reason": "str", "index": "int", "logprobs": _LOGPROBS, "message": _MSG}, None)
_CTD = ("obj", {"text_tokens": "int", "accepted_prediction_tokens": "int", "audio_tokens": "int", "reasoning_tokens": ("int", "reasoning"),
                "rejected_prediction_tokens": "int"}, "ctd")
_PTD = ("obj", {"text_tokens": "int", "audio_tokens": "int", "cached_tokens": ("int", "cached"), "cache_creation_input_tokens": ("int", "creation")}, "ptd")
_USAGE = ("obj", {"prompt_tokens": ("int", "in"), "completion_tokens": ("int", "out"), "total_tokens": ("int", "total"),
                  "completion_tokens_details": _CTD, "prompt_tokens_details": _PTD}, "usage")
CHAT = ("obj", {"id": "str", "choices": ("arr", _CHOICE), "created": "created", "model": ("str", "model"), "service_tier": "str",
                "system_fingerprint": "str", "object": "str", "usage": _USAGE, "obfuscation": "str"}, None)
EMBEDDINGS = ("obj", {"object": "str", "data": ("arr", ("obj", {"object": "str", "embedding": ("strobj", ("arr", "float")), "index": "int"}, None)),
                      "model": ("str", "model"), "usage": ("obj", {"prompt_tokens": ("int", "in"), "total_tokens": ("int", "total")}, "usage")}, None)
_CM_LOGPROBS = ("obj", {"tokens": ("arr", "str"), "token_logprobs": ("arr", "float"), "top_logprobs": ("arr", ("map", "float")),
                        "text_offset": ("arr", "int")}, None)
COMPLETIONS = ("obj", {"id": "str", "object": "str", "created": "created", "model": ("str", "model"), "system_fingerprint": "str",
                       "choices": ("arr", ("obj", {"text": "str", "index": "int", "logprobs": _CM_LOGPROBS, "finish_reason": "str"}, None)),
                       "usage": _USAGE}, None)
SCHEMA = {"chat": CHAT, "embeddings": EMBEDDINGS, "completions": COMPLETIONS, "responses": R.RESPONSE, "rerank": Q.RESPONSE}
TRAILING = {"chat": True, "embeddings": True, "completions": False, "responses": True, "rerank": True}
# the /v1/responses root's members from the 33rd of the kernel's table on: repeats are not tracked
UNTRACKED = {id(R.RESPONSE[1]): {"presence_penalty", "frequency_penalty", "store"}}


class _Out(R._Out):
    def __init__(self, rule):
        super().__init__(rule)
        self.rule = rule


class _PredMixin:
    """_Walk plus the library's decline rules named, base64 members, untracked repeats and the raw value of every captured int"""
    def value(self, i, t, depth):
        p = self.p
        i0 = R._ws(p, i)
        if t == "b64":   # []byte: null, or base64.StdEncoding text; an escape or a control byte is not restated
            if i0 < len(p) and p[i0] == 0x6E:
                return super().value(i, "str", depth)
            if i0 >= len(p) or p[i0] != 0x22:
                raise R._Fail
            j, raw, esc = R._string(p, i0)
            if esc:
                raise _Out("esc_b64")
            if len(raw) % 4:
                raise R._Fail
            for k, ch in enumerate(raw):
                if ch < 0x20:
                    raise _Out("ctl_b64")
                if not (chr(ch).isascii() and (chr(ch).isalnum() or ch in b"+/" or (ch == 0x3D and k >= len(raw) - 2))):
                    raise R._Fail
            if len(raw) >= 2 and raw[-2] == 0x3D and raw[-1] != 0x3D:
                raise R._Fail
            return j
        if isinstance(t, tuple) and t[0] == "obj" and i0 < len(p) and p[i0] == 0x7B:
            return self._obj(i0, t, depth)
        if isinstance(t, tuple) and t[0] == "arr" and depth >= R.MAX_TYPED_DEPTH and i0 < len(p) and p[i0] == 0x5B and R._ws(p, i0 + 1) < len(p) and p[R._ws(p, i0 + 1)] != 0x5D:
            raise _Out("typed_depth")
        if t == "any":
            try:
                return super().value(i, t, depth)
            except R._Out:
                raise _Out("skip_depth")
        if isinstance(t, tuple) and t[0] == "str" and t[1] == "model":
            if i0 < len(p) and p[i0] == 0x22 and R._string(p, i0)[2]:
                raise _Out("esc_model")
        try:
            j = super().value(i, t, depth)
        except _Out:
            raise
        except R._Out as e:
            raise _Out("f64" if self.kind == "rerank" else "union" if not isinstance(e, _Out) else e.rule)
        if isinstance(t, tuple) and t[0] == "int" and t[1] and p[i0] != 0x6E:
            self.raw[t[1]] = int(p[i0:j])
        return j

    def _obj(self, i, t, depth):
        p = self.p
        if t[2]:
            self.caps[t[2]] = True
        i = R._ws(p, i + 1)
        if i < len(p) and p[i] == 0x7D:
            return i + 1
        if depth >= R.MAX_TYPED_DEPTH:
            raise _Out("typed_depth")
        seen, untracked = set(), UNTRACKED.get(id(t[1]), ())
        while True:
            if i >= len(p) or p[i] != 0x22:
                raise R._Fail
            j, key, esc = R._string(p, i)
            if esc:
                raise _Out("esc_key")
            i = R._ws(p, j)
            if i >= len(p) or p[i] != 0x3A:
                raise R._Fail
            k = key.decode("latin-1")
            if k in t[1] and k not in untracked:
                if k in seen:
                    raise _Out("dup_key")
                seen.add(k)
            i = R._ws(p, self.value(i + 1, t[1].get(k, "any"), depth + 1))
            if i >= len(p):
                raise R._Fail
            if p[i] == 0x2C:
                i = R._ws(p, i + 1)
                continue
            if p[i] == 0x7D:
                return i + 1
            raise R._Fail


class _Pred(_PredMixin, R._Walk):
    pass


class _RerankPred(_PredMixin, Q._RerankWalk):
    pass


def predict(kind, body):
    """→ (verdict OK / FAIL / OUT, rule of an OUT or None, captures, raw captured ints)"""
    w = (_RerankPred if kind == "rerank" else _Pred)(body)
    w.kind, w.raw = kind, {}
    try:
        e = w.value(0, SCHEMA[kind], 0)
        if not TRAILING[kind] and R._ws(body, e) != len(body):
            raise R._Fail
    except R._Fail:
        return R.FAIL, None, w.caps, w.raw
    except _Out as x:
        return R.OUT, x.rule, w.caps, w.raw
    if kind == "completions" and w.caps.get("usage") and any(not 0 <= v < 1 << 31 for v in w.raw.values()):
        return R.OUT, "big", w.caps, w.raw
    return R.OK, None, w.caps, w.raw


def _u7(vals, mask):
    """(input, cached, cache_creation, output, total, reasoning) with the mask bits of aigw_usage → the record's usage 7-tuple"""
    bits = (1, 8, 16, 2, 4, 32)
    return tuple(v if mask & b else 0 for v, b in zip(vals, bits)) + (mask,)


def _oracle_cpp(kind, body):
    """(ok, usage 7-tuple, model) of the C++ oracle"""
    ok, u, m = {"chat": O.response_openai, "embeddings": O.response_embeddings, "completions": O.response_completions}[kind](body)
    if kind == "embeddings":
        return ok, (u.input, 0, 0, 0, u.total, 0, 5), m
    return ok, _u7((u.input, u.cached, u.cache_creation, u.output, u.total, u.reasoning), u.mask), m


def expect(kind, body):
    """the record the GPU must return: (status, usage 7-tuple, model bytes, decline rule or None)"""
    v, rule, caps, _ = predict(kind, body)
    if v == R.OUT:
        return DECLINED, ZERO7, b"", rule
    if v == R.FAIL:
        return INTERNAL, ZERO7, b"", None
    if kind in ("chat", "embeddings", "completions"):
        ok, u, m = _oracle_cpp(kind, body)
        assert ok, (kind, body[:200])   # held by test_predict_agrees_with_the_cpp_oracle
        return OK, u, m, None
    if kind == "responses":
        u = _u7((caps.get("in", 0), caps.get("cached", 0), caps.get("creation", 0), caps.get("out", 0), caps.get("total", 0), caps.get("reasoning", 0)),
                63 if caps.get("usage") else 0)
        return OK, u, caps.get("model", b""), None
    if not caps.get("tokens"):
        return OK, ZERO7, b"", None
    inp, out = caps.get("in"), caps.get("out")
    mask = 4 | (1 if inp is not None else 0) | (2 if out is not None else 0)
    return OK, _u7((inp or 0, 0, 0, out or 0, ((inp or 0) + (out or 0)) & 0xFFFFFFFF, 0), mask), b"", None


# ---------------------------------------------------------------- reference models of the kernels' number conversions
def parse_i64_model(text):
    """strconv.ParseInt(text, 10, 64) then uint32(): the low 32 bits, or None when it fails (fraction, exponent, leading zero,
    overflow).  What tjson.cuh's scan_number + parse_i64 compute."""
    s = text.decode("latin-1")
    d = s[1:] if s.startswith("-") else s
    if not d.isdigit() or not d.isascii() or (len(d) > 1 and d[0] == "0"):
        return None
    v = int(s)
    if not -(1 << 63) <= v < 1 << 63:
        return None
    return v & 0xFFFFFFFF


def f64_trunc_u32_model(text):
    """uint32(float64(text)) as Go computes it (ParseFloat is correctly rounded, as Python's float), or None where the rounded
    value lies outside (-1, 2^32) and the conversion is implementation-defined"""
    f = float(text)
    return int(f) if -1.0 < f < 4294967296.0 else None


# ---------------------------------------------------------------- corpora
INT_TEXTS = [b"0", b"-0", b"1", b"2147483647", b"2147483648", b"4294967295", b"4294967296", b"4294967297", b"9223372036854775807",
             b"9223372036854775808", b"-1", b"-9223372036854775808", b"-9223372036854775809", b"12345678901234567890", b"123456789012345678901",
             b"01", b"1.0", b"1e0", b"1E+0", b"null"]
COUNTERS = {   # kind → counter positions: (usage path, member)
    "chat": [((), "prompt_tokens"), ((), "completion_tokens"), ((), "total_tokens"), (("prompt_tokens_details",), "cached_tokens"),
             (("prompt_tokens_details",), "cache_creation_input_tokens"), (("completion_tokens_details",), "reasoning_tokens")],
    "embeddings": [((), "prompt_tokens"), ((), "total_tokens")],
    "responses": [((), "input_tokens"), ((), "output_tokens"), ((), "total_tokens"), (("input_tokens_details",), "cached_tokens"),
                  (("input_tokens_details",), "cache_creation_input_tokens"), (("output_tokens_details",), "reasoning_tokens")],
    "rerank": [(("tokens",), "input_tokens"), (("tokens",), "output_tokens")],
}
COUNTERS["completions"] = COUNTERS["chat"]


def base(kind, usage=None, model=b'"gpt-4o"'):
    """a small valid body of the kind whose usage object is `usage` (raw bytes, or None for none) and model `model` (raw)"""
    u = b"" if usage is None else b',"usage":' + usage
    if kind == "chat":
        return b'{"id":"c1","object":"chat.completion","created":1,"model":' + model + b',"choices":[{"index":0,"message":{"role":"assistant","content":"hi"},"finish_reason":"stop"}]' + u + b"}"
    if kind == "embeddings":
        return b'{"object":"list","data":[{"object":"embedding","index":0,"embedding":[0.5,-1]}],"model":' + model + u + b"}"
    if kind == "completions":
        return b'{"id":"c1","object":"text_completion","created":1,"model":' + model + b',"choices":[{"text":"hi","index":0,"logprobs":null,"finish_reason":"stop"}]' + u + b"}"
    if kind == "responses":
        return b'{"id":"r1","object":"response","created_at":1,"status":"completed","model":' + model + b',"output":[{"type":"message","id":"m","status":"completed","role":"assistant","content":[{"type":"output_text","text":"hi","annotations":[]}]}]' + u + b"}"
    return b'{"id":"q1","results":[{"index":0,"relevance_score":0.5}],"meta":{"api_version":{"version":"2"}' + (b',"tokens":' + usage if usage is not None else b"") + b"}}"


def _usage_with(kind, path, member, text):
    """a usage object of the kind with `member` (under the sub-object `path`) set to the raw `text`, other counters small"""
    if kind == "rerank":
        other = "output_tokens" if member == "input_tokens" else "input_tokens"
        return b'{"' + member.encode() + b'":' + text + b',"' + other.encode() + b'":3}'
    top = {"prompt_tokens": b"11", "completion_tokens": b"22", "total_tokens": b"33"} if kind != "responses" else {"input_tokens": b"11", "output_tokens": b"22", "total_tokens": b"33"}
    if kind == "embeddings":
        top = {"prompt_tokens": b"11", "total_tokens": b"33"}
    parts = []
    for k, v in top.items():
        parts.append(b'"%s":%s' % (k.encode(), text if (not path and k == member) else v))
    if path:
        parts.append(b'"%s":{"%s":%s}' % (path[0].encode(), member.encode(), text))
    return b"{" + b",".join(parts) + b"}"


def integer_corpus():
    out = []
    for kind in KINDS:
        for path, member in COUNTERS[kind]:
            for t in INT_TEXTS:
                out.append((kind, "int", base(kind, _usage_with(kind, path, member, t))))
    return out


def _float_texts():
    """rerank float counters at f64_trunc_u32's edges"""
    ts = []
    for k in range(33):
        for I in (2 ** k - 1, 2 ** k, 2 ** k + 1):
            ts += [b"%d" % I, b"%d.0" % I, b"-%d" % I if I <= 1 else b"%d.5" % I]
    for I in (0, 1, 3, 1000, 2 ** 20 + 1, 2 ** 31 - 1, 2 ** 32 - 2, 2 ** 32 - 1):
        q = 54 if I == 0 else 53 - (I.bit_length() - 1)
        tie = 10 ** q - 5 ** q                               # 1 - 2^-q written out with q decimals
        for f in (tie - 1, tie, tie + 1):
            ts.append(b"%d.%0*d" % (I, q, f))
            ts.append(b"%d.%0*d7" % (I, q, f))               # a digit past the q-th
        ts.append(b"-%d.%0*d" % (I, q, tie) if I == 0 else b"%d.%s" % (I, b"9" * q))
    for L in (37, 38, 39, 53, 54, 55):
        for I in (0, 1, 2 ** 31 - 1):
            ts += [b"%d.%s" % (I, b"9" * L), b"%d.%s8" % (I, b"9" * (L - 1)), b"%d.%s" % (I, b"9" * (L - 1) + b"5")]
    for d in (10, 11, 308, 309):
        ts += [b"1" + b"0" * (d - 1), b"4" + b"2" * (d - 1), b"-1" + b"0" * (d - 1), b"9" * d + b".5"]
    ts += [b"-0.99999999999999994", b"-0.99999999999999995", b"-1", b"-0", b"-0.0", b"1e0", b"1E+2", b"0.1e1", b"null", b'"1"', b"4294967295.999999999"]
    return list(dict.fromkeys(ts))


def float_corpus():
    return [("rerank", "f64", base("rerank", b'{"input_tokens":' + t + b',"output_tokens":' + (b"2" if i % 2 else t) + b"}")) for i, t in enumerate(_float_texts())]


NEST_DEPTHS = (63, 64, 65, 512, 513, 4096)
RULES = ("esc_key", "dup_key", "typed_depth", "skip_depth", "esc_model", "big", "f64", "union")


def _nest(d, mode):
    """a value that opens d containers: arrays, objects, or the two alternating"""
    opens, closes = [], []
    for k in range(d):
        obj = mode == "obj" or (mode == "alt" and k % 2)
        opens.append(b'{"k":' if obj else b"[")
        closes.append(b"}" if obj else b"]")
    return b"".join(opens) + b"1" + b"".join(reversed(closes))


def nesting_corpus():
    out = []
    for kind in KINDS:
        for d in NEST_DEPTHS:
            for mode in ("arr", "obj", "alt"):
                v = _nest(d, mode)
                b = base(kind, None)
                out.append((kind, "nest_root", b[:-1] + b',"x":' + v + b"}"))
                if kind != "rerank":
                    out.append((kind, "nest_usage", base(kind, _usage_with(kind, (), "total_tokens", b"5")[:-1] + b',"x":' + v + b"}")))
                else:
                    out.append((kind, "nest_usage", base(kind, b'{"input_tokens":1,"x":' + v + b"}")))
                if kind == "chat":
                    out.append((kind, "nest_message", b.replace(b'"content":"hi"', b'"content":"hi","x":' + v)))
        # known members at document depth 11, 12 and 13 below an unknown member: skipped, never captured
        for d in (11, 12, 13):
            inner = b'{"usage":' + _usage_with(kind, (), COUNTERS[kind][0][1], b"7") + b',"model":"deep"}'
            out.append((kind, "known_deep", base(kind, None)[:-1] + b',"x":' + b"[" * (d - 2) + inner + b"]" * (d - 2) + b"}"))
        out.append((kind, "typed_deepest", DEEPEST[kind]))
    return out


# The five schemas do not recurse: their deepest typed container sits at depth 9 (chat, /v1/responses), 5 (completions), 3
# (embeddings) or 2 (rerank), so walk's MAXD = 12 cannot be reached by a buffered response and "typed_depth" never occurs here.
# These bodies fill each schema's deepest typed path.
DEEPEST = {
    "chat": b'{"choices":[{"logprobs":{"content":[{"top_logprobs":[{"bytes":[1,2]}]}],"refusal":null},"message":{"reasoning_content":{"reasoningContent":{"reasoningText":{"text":"t"},"redactedContent":"QUJD"}}}}],"usage":{"prompt_tokens":1}}',
    "embeddings": b'{"data":[{"embedding":[1,2.5,-3e2]},{"embedding":"AAAA"}],"usage":{"prompt_tokens":1,"total_tokens":2}}',
    "completions": b'{"choices":[{"logprobs":{"top_logprobs":[{"a":1.5,"b":-2}],"text_offset":[0,1],"tokens":["a"]}}],"usage":{"prompt_tokens":1,"completion_tokens":2,"total_tokens":3}}',
    "responses": b'{"output":[{"type":"message","content":[{"type":"output_text","text":"t","annotations":[{"type":"url_citation","url":"u","title":"t","start_index":0,"end_index":1}],"logprobs":[{"token":"a","logprob":-1,"bytes":[97],"top_logprobs":[{"token":"a","bytes":[97],"logprob":-1}]}]}]}],"usage":{"input_tokens":1}}',
    "rerank": b'{"results":[{"index":1,"relevance_score":0.25},null],"meta":{"tokens":{"input_tokens":4,"output_tokens":5}}}',
}


def keys_corpus():
    out = []
    for kind in KINDS:
        member = COUNTERS[kind][0][1]
        b = base(kind, _usage_with(kind, (), member, b"7"))
        key = b'"tokens"' if kind == "rerank" else b'"usage"'
        for alt in (key.upper(), key[:2].upper() + key[2:], key[:-2] + b'"', key[:-1] + b'_"', b'"\\u00%x' % key[1] + key[2:]):
            out.append((kind, "key_variant", b.replace(key + b":", alt + b":", 1)))
        out.append((kind, "key_variant", b.replace(b'"%s"' % member.encode(), b'"\\u00%x%s"' % (ord(member[0]), member[1:].encode()), 1)))
        k0 = b.index(key + b":")
        out.append((kind, "key_repeat", b[:k0] + key + b':{},' + b[k0:]))
        out.append((kind, "key_repeat", b.replace(b'"%s":7' % member.encode(), b'"%s":7,"%s":8' % (member.encode(), member.encode()), 1)))
        for k in (30, 31, 32):   # the captured member after 30, 31 or 32 unknown ones
            pad = b"".join(b'"u%d":%d,' % (x, x) for x in range(k))
            out.append((kind, "key_position", b.replace(key + b":{", key + b":{" + pad, 1)))
    # /v1/responses: the root's members from the 33rd of the kernel's table on are not tracked for repeats; the 32nd is
    r = base("responses", _usage_with("responses", (), "input_tokens", b"7"))
    out += [("responses", "union", r.replace(b'"output":[', b'"output":[{"type":"web_search_call","id":"w"},', 1)), ("responses", "union", r[:-1] + b',"presence_penalty":1e2}'),
            ("responses", "union", r[:-1] + b',"tools":[{"type":"mcp"}]}'), ("responses", "union", r.replace(b'{"type":"message"', b'{"t\\u0079pe":"message","type":"message"', 1))]
    for m, v in ((b"store", b"true"), (b"presence_penalty", b"0.5"), (b"frequency_penalty", b"1"), (b"user", b'"x"'), (b"truncation", b'"auto"')):
        out.append(("responses", "key_repeat", r[:-1] + b',"%s":%s,"%s":%s}' % (m, v, m, v)))
    return out


def model_corpus():
    out = []
    for kind in KINDS:
        u = _usage_with(kind, (), COUNTERS[kind][0][1], b"9")
        for m in (b'""', b"null", b'"a\\u0062"', b'"a\\"b"', b'"' + b"m" * 4096 + b'"', '"cafè 東京"'.encode(), b'"\\/"', b"5", b'"\x01\xff"'):
            out.append((kind, "model", base(kind, u, model=m)))
        b = base(kind, u)
        for tail in (b" ", b"\n\t \r", b"x", b"{}", b"}", b" null", b"\x00", b'{"usage":{}}'):
            out.append((kind, "trailing", b + tail))
        for lead in (b" ", b"\n\t"):
            out.append((kind, "leading", lead + b))
    return out


def _gold(name, key):
    return [c["body"].encode() for c in json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", name), encoding="utf-8"))[key]]


def seeds(kind):
    """15-25 bodies the kind decodes: its goldens, the existing generators and the edge corpora"""
    gold = {"chat": [b for b in RG._bodies(7, 60) if O.response_openai(b)[0]][:12], "completions": _gold("completions_cases.json", "buffered"),
            "responses": _gold("responses_cases.json", "buffered"), "rerank": _gold("rerank_cases.json", "response_body"), "embeddings": []}[kind]
    own = [b for k, _, b in integer_corpus()[::5] + keys_corpus() + model_corpus()[::3] if k == kind and len(b) < 1500] + [DEEPEST[kind]]
    out = [b for b in gold + own if expect(kind, b)[0] == OK]
    return list(dict.fromkeys(out))[:22]


MUTANTS_PER_KIND = 20000


def mutation_corpus(kind):
    """one-byte deletions, duplications and replacements (MUT_BYTES) of the kind's seeds, sampled to MUTANTS_PER_KIND"""
    rng = random.Random("response-usage-" + kind)
    cands = []
    for s in seeds(kind):
        for i in range(len(s)):
            cands.append(s[:i] + s[i + 1:])
            cands.append(s[:i + 1] + s[i:])
            cands += [s[:i] + bytes([c]) + s[i + 1:] for c in MUT_BYTES if c != s[i]]
    cands = sorted(set(cands) - set(seeds(kind)))
    rng.shuffle(cands)
    return cands[:MUTANTS_PER_KIND]


def edge_corpus():
    """(kind, label, body) for every hand-built edge above"""
    return integer_corpus() + float_corpus() + nesting_corpus() + keys_corpus() + model_corpus()


# ---------------------------------------------------------------- CEL: a big-integer model of the compiled subset
I64 = (-(1 << 63), (1 << 63) - 1)
TOKS = ("input_tokens", "cached_input_tokens", "cache_creation_input_tokens", "output_tokens", "total_tokens", "reasoning_tokens")
CMP = ("==", "!=", "<", "<=", ">", ">=")


class CelModel:
    """Parses the subset aigw_cost_compile accepts and evaluates it on exact integers.  A value is (error class, value, type); && and
    || absorb an error when the other side decides, ?: evaluates only the taken branch, and an error otherwise propagates (the left
    operand's first).  rc: 0, or 2 when NewProgram's sanity evaluation (zero counters, "dummy" strings) fails or is not an integer."""
    LEVELS = (("||",), ("&&",), ("==", "!=", "<=", ">=", "<", ">"), ("+", "-"), ("*", "/", "%"))

    def __init__(self, expr):
        self.s, self.i = expr, 0
        self.tree = self._cond()
        self._ws()
        assert self.i == len(self.s), expr
        e, v, t = self._ev(self.tree, dict(dict.fromkeys(TOKS, 0), model="dummy", backend="dummy", route_name="dummy"))
        self.rc = 2 if e or t not in "iu" or (t == "i" and v < 0) else 0

    def _ws(self):
        while self.i < len(self.s) and self.s[self.i] in " \t\r\n":
            self.i += 1

    def _at(self, w):
        self._ws()
        if not self.s.startswith(w, self.i) or (w in ("<", ">", "!") and self.s.startswith(w + "=", self.i)):
            return False
        self.i += len(w)
        return True

    def _cond(self):
        c = self._bin(0)
        if not self._at("?"):
            return c
        a = self._bin(0)
        assert self._at(":")
        return ("?", c, a, self._cond())

    def _bin(self, lvl):
        if lvl == len(self.LEVELS):
            return self._unary()
        l = self._bin(lvl + 1)
        while True:
            op = next((o for o in self.LEVELS[lvl] if self._at(o)), None)
            if op is None:
                return l
            l = (op, l, self._bin(lvl + 1))

    def _unary(self):
        if self._at("!"):
            return ("!", self._unary())
        if self._at("-"):
            return ("neg", self._unary())
        self._ws()
        s, i = self.s, self.i
        if s[i] == "(":
            self.i += 1
            e = self._cond()
            assert self._at(")")
            return e
        if s[i] in "'\"":
            j = s.index(s[i], i + 1)
            self.i = j + 1
            return ("lit", 0, s[i + 1:j], "s")
        j = i
        while j < len(s) and (s[j].isalnum() or s[j] == "_"):
            j += 1
        w, self.i = s[i:j], j
        if w[0].isdigit():
            return ("lit", 0, int(w[:-1], 0), "u") if w[-1] in "uU" else ("lit", 0, int(w, 0), "i")
        if w in ("true", "false"):
            return ("lit", 0, int(w == "true"), "b")
        if w in ("int", "uint"):
            assert self._at("(")
            a = self._cond()
            assert self._at(")")
            return (w, a)
        return ("var", w)

    def eval(self, model, backend, route, *tok):
        """→ (error class, cost) as EvaluateProgram returns them; 5: an int result below zero"""
        e, v, t = self._ev(self.tree, dict(zip(TOKS, tok), model=model, backend=backend, route_name=route))
        if e:
            return e, 0
        return (5, 0) if t == "i" and v < 0 else (0, v)

    def _ev(self, n, env):
        k = n[0]
        if k == "lit":
            return n[1:]
        if k == "var":
            v = env[n[1]]
            return (0, v, "s") if isinstance(v, str) else (0, v, "u")
        if k == "?":
            c = self._ev(n[1], env)
            return c if c[0] else self._ev(n[2] if c[1] else n[3], env)
        if k in ("&&", "||"):
            a, b = self._ev(n[1], env), self._ev(n[2], env)
            dom = 0 if k == "&&" else 1
            if (not a[0] and a[1] == dom) or (not b[0] and b[1] == dom):
                return 0, dom, "b"
            return (a[0] or b[0]), (0 if a[0] or b[0] else 1 - dom), "b"
        if k in ("!", "neg", "int", "uint"):
            e, v, _ = self._ev(n[1], env)
            t = {"!": "b", "neg": "i", "int": "i", "uint": "u"}[k]
            if e:
                return e, 0, t
            r = {"!": 1 - v, "neg": -v, "int": v, "uint": v}[k]
            if t == "i" and not I64[0] <= r <= I64[1]:
                return 1, 0, t
            if t == "u" and r < 0:
                return 2, 0, t
            return 0, r, t
        a, b = self._ev(n[1], env), self._ev(n[2], env)
        t = "b" if k in CMP else a[2]
        if a[0] or b[0]:
            return (a[0] or b[0]), 0, t
        x, y = a[1], b[1]
        if k in CMP:
            return 0, int({"==": x == y, "!=": x != y, "<": x < y, "<=": x <= y, ">": x > y, ">=": x >= y}[k]), t
        if k in "/%" and y == 0:
            return (3 if k == "/" else 4), 0, t
        if k == "/":
            r = abs(x) // abs(y) * (1 if (x < 0) == (y < 0) else -1)   # Go: truncated toward zero
        elif k == "%":
            r = abs(x) % abs(y) * (1 if x >= 0 else -1)                 # Go: the sign of the dividend
            if t == "i" and x == I64[0] and y == -1:
                r = 1 << 63                                                # MinInt64 % -1 overflows in cel-go, as MinInt64 / -1
        else:
            r = {"+": x + y, "-": x - y, "*": x * y}[k]
        if t == "i":
            return (0, r, t) if I64[0] <= r <= I64[1] else (1, 0, t)
        return (0, r, t) if 0 <= r < 1 << 64 else (2, 0, t)


def cel_random_corpus():
    """the expressions, rows and models of test_cel_gpu.test_random_expressions_match_oracle"""
    rng = np.random.default_rng(11)
    rows = [(0, 0, 0, 0, 0, 0), (1, 0, 0, 1, 2, 0), (200, 100, 1, 2, 3, 0), (4294967295,) * 6, (100, 0, 0, 2000, 3, 0), (7, 3, 2, 5, 12, 1)] + \
           [tuple(int(x) for x in rng.integers(0, 2**32, 6)) for _ in range(10)] + [tuple(int(x) for x in rng.integers(0, 50, 6)) for _ in range(16)]
    models = [["gpt-4o", "cool_model", "", "aws"][i % 4] for i in range(len(rows))]
    exprs = [CG.gen(rng, "ui"[int(rng.integers(0, 2))], int(rng.integers(1, 5))) for _ in range(40 * 8)]
    return exprs, rows, models


# Operands of the boundary table, as CEL text.  Each is gated on input_tokens, so that NewProgram's sanity evaluation (zero counters)
# sees 1 and a record whose counters are all 2^32 - 1 sees the operand; the counters themselves reach the VM through C_PUSH_TOK.
INT_OPERANDS = ["0", "1", "-1", "2147483648", "4294967295", "4294967296", "4611686018427387904", "9223372036854775807", "-9223372036854775807 - 1",
                "int(input_tokens)", "7", "1317624576693539401"]   # 7 * 1317624576693539401 = 2^63 - 1
UINT_OPERANDS = ["0u", "1u", "2147483648u", "4294967295u", "4294967296u", "4611686018427387904u", "9223372036854775807u", "9223372036854775808u",
                 "18446744073709551614u", "18446744073709551615u", "input_tokens"]
MAXTOK = (4294967295,) * 6


def gate(text, ty, other=None):
    return "(input_tokens == 4294967295u ? (%s) : %s)" % (text, other or ("1" if ty == "i" else "1u"))


def cel_boundary_exprs():
    """+ - * / % over every ordered pair of operands of one type, unary -, int() and uint(), and sums that land exactly on 2^63 - 1
    and 2^64 - 1 and one past them"""
    out = []
    for ty, ops in (("i", INT_OPERANDS), ("u", UINT_OPERANDS)):
        for op in "+-*/%":
            out += ["%s %s %s" % (gate(a, ty), op, gate(b, ty)) for a in ops for b in ops]
    out += ["-%s" % gate(a, "i", "-1") for a in INT_OPERANDS] + ["uint(%s)" % gate(a, "i") for a in INT_OPERANDS] + ["int(%s)" % gate(a, "u") for a in UINT_OPERANDS]
    out += ["%s * 1317624576693539401 + 0" % gate("7", "i"), "%s * 1317624576693539401 + %s" % (gate("7", "i"), gate("1", "i")),
            "18446744073709551614u + input_tokens / 4294967295u", "18446744073709551615u + input_tokens / 4294967295u",
            "input_tokens * output_tokens", "input_tokens * output_tokens * 2u", "input_tokens * output_tokens + 8589934590u", "input_tokens * output_tokens + 8589934591u",
            "%s / -1" % gate("-9223372036854775807 - 1", "i"), "%s %% -1" % gate("-9223372036854775807 - 1", "i")]
    return out


# truth tables: true, false, and two bools that fail only when the counters are 2^32 - 1 (uint overflow, class 2; division by zero, 3)
BOOLS = {"T": "true", "F": "false", "E2": "(input_tokens == 0u || 0u - input_tokens == 1u)", "E3": "(input_tokens == 0u || 1u / (output_tokens - output_tokens) == 1u)"}
INTS = {"1": "1", "2": "2", "E1": "(input_tokens == 0u ? 0 : 9223372036854775807 + int(input_tokens))", "E3": "(input_tokens == 0u ? 0 : 1 / int(output_tokens - output_tokens))"}


def cel_truth_exprs():
    out = ["(%s %s %s) ? 1 : 2" % (BOOLS[a], op, BOOLS[b]) for a in BOOLS for b in BOOLS for op in ("&&", "||")]
    return out + ["%s ? %s : %s" % (BOOLS[c], INTS[x], INTS[y]) for c in BOOLS for x in INTS for y in INTS]


# ================================================================ self-checks
def test_predict_agrees_with_the_cpp_oracle():
    """wherever predict says OK or FAIL for chat, embeddings and completions the C++ oracle agrees, with the walk's model on OK"""
    n = collections.Counter()
    for kind in ("chat", "embeddings", "completions"):
        for b in [b for k, _, b in edge_corpus() if k == kind] + mutation_corpus(kind)[:5000]:
            v, _, caps, _ = predict(kind, b)
            if v == R.OUT:
                continue
            ok, _, m = _oracle_cpp(kind, b)
            assert ok == (v == R.OK), (kind, b[:300], v)
            if ok:
                assert m == caps.get("model", b""), (kind, b[:300])
            n[kind, v] += 1
    assert all(n[k, v] > 100 for k in ("chat", "embeddings", "completions") for v in (R.OK, R.FAIL)), n


def test_integer_counters_follow_parse_i64():
    """each counter text in each integer position: the low 32 bits where ParseInt accepts it (completions: a decline outside
    [0, 2^31)), INTERNAL where it does not, and null leaves the counter unset"""
    seen = set()
    for kind, _, b in integer_corpus():
        if kind == "rerank":
            continue   # float64 counters: test_rerank_float_counters
        st, u, _, rule = expect(kind, b)
        ub = b[b.index(b'"usage"'):]
        t = next(t for t in INT_TEXTS if b":" + t + b"," in ub or b":" + t + b"}" in ub)
        want = parse_i64_model(t)
        if t == b"null":
            assert st == OK, (kind, b)
        elif want is None:
            assert st == INTERNAL, (kind, b)
        elif kind == "completions" and not 0 <= int(t) < 1 << 31:
            assert (st, rule) == (DECLINED, "big"), (kind, b)
        else:
            assert st == OK and want in u[:6], (kind, b, u)
        seen.add((kind, t))
    assert len(seen) == 4 * len(INT_TEXTS)
    assert [parse_i64_model(t) for t in (b"-1", b"4294967296", b"-9223372036854775808", b"9223372036854775808", b"-0", b"01")] == [0xFFFFFFFF, 0, 0, None, 0, None]


def test_rerank_float_counters():
    """the float texts reach every branch of f64_trunc_u32: rounding up to I + 1 (the tie and above), staying at I (one below the
    tie), declines outside (-1, 2^32), and the exponent / 309-digit declines; each record is int(float(text))"""
    seen = collections.Counter()
    for _, _, b in float_corpus():
        st, u, _, rule = expect("rerank", b)
        t = b[b.index(b'"input_tokens":') + 15:b.index(b',"output_tokens"')]
        if st == OK:
            want = None if t == b"null" else f64_trunc_u32_model(t)
            assert (u[0] if u[6] & 1 else None) == want, (t, u)
            ip = t.split(b".")[0]
            seen["up" if b"." in t and want == int(ip) + 1 else "ok"] += 1
        elif st == DECLINED:
            assert rule == "f64", (t, rule)
            if b"e" not in t.lower() and len(t.lstrip(b"-").split(b".")[0]) <= 308:
                assert f64_trunc_u32_model(t) is None, t
                seen["out_of_range"] += 1
            else:
                seen["unrestated"] += 1
        else:
            assert t == b'"1"', t
            seen["fail"] += 1
    assert seen["up"] >= 20 and seen["ok"] >= 150 and seen["out_of_range"] >= 10 and seen["unrestated"] >= 4, seen
    # the model's own edges: the tie rounds up to the even I + 1, one unit below it stays at I
    assert f64_trunc_u32_model(b"0." + b"9" * 17) == 1 and f64_trunc_u32_model(b"4294967294." + b"9" * 22) == 4294967295
    assert f64_trunc_u32_model(b"4294967295.9999999") is None and f64_trunc_u32_model(b"-0.99999999999999994") == 0


def test_every_rule_and_edge_occurs():
    """every decline rule (but typed_depth, unreachable: see DEEPEST) occurs; skipped nesting of 63 and 64 levels decodes and of 65,
    512, 513 and 4096 levels declines, never INTERNAL; trailing bytes fail completions only"""
    recs = [(k, lbl, b, expect(k, b)) for k, lbl, b in edge_corpus()]
    rules = collections.Counter(r[3] for _, _, _, r in recs if r[0] == DECLINED)
    print("\nedge corpus decline rules:", dict(rules))
    assert all(rules[x] > 0 for x in RULES if x != "typed_depth"), rules
    by = collections.Counter((k, lbl) for k, lbl, _, _ in recs)
    for kind in KINDS:
        assert by[kind, "int"] == len(COUNTERS[kind]) * len(INT_TEXTS) and by[kind, "nest_root"] == 3 * len(NEST_DEPTHS) and by[kind, "known_deep"] == 3
    assert all(r[0] in (OK, DECLINED) for _, lbl, _, r in recs if lbl.startswith("nest_"))
    nest = [r[0] for _, lbl, _, r in recs if lbl == "nest_root"]
    assert nest.count(DECLINED) == 4 * 3 * len(KINDS) and nest.count(OK) == 2 * 3 * len(KINDS), collections.Counter(nest)
    assert all(r[0] == OK for _, lbl, _, r in recs if lbl in ("known_deep", "typed_deepest")), [(k, b[:80], r) for k, lbl, b, r in recs if lbl in ("known_deep", "typed_deepest") and r[0] != OK]
    trail = collections.Counter((k, r[0]) for k, lbl, b, r in recs if lbl == "trailing" and b.rstrip(b" \t\r\n") == b)
    assert trail["completions", OK] == 0 and all(trail[k, INTERNAL] == 0 for k in KINDS if k != "completions"), trail
    ws = [(k, r[0]) for k, lbl, b, r in recs if lbl in ("trailing", "leading") and b.strip(b" \t\r\n") != b]
    assert all(st == OK for _, st in ws), ws


def test_mutation_corpora_are_pinned():
    """15-25 seeds per kind, all decoded; 20 000 mutants per kind; the corpora reproducible (hash pinned)"""
    h = hashlib.sha256()
    for kind in KINDS:
        s = seeds(kind)
        assert 15 <= len(s) <= 25, (kind, len(s))
        m = mutation_corpus(kind)
        assert len(m) == MUTANTS_PER_KIND
        for b in s + m:
            h.update(kind.encode() + len(b).to_bytes(4, "little") + b)
    assert h.hexdigest() == MUTATION_SHA256, h.hexdigest()


MUTATION_SHA256 = "1747d835c7270c53f3a1032b0a206a1a75506e4db71bb0eaf94fadd2a24992e9"


def test_cel_model_agrees_with_the_oracle():
    """the big-integer model against O.Cel: the random corpus of test_cel_gpu (compile verdict and every evaluation), the boundary
    table and the truth tables (with counters at 2^32 - 1, where every error class occurs)"""
    exprs, rows, models = cel_random_corpus()
    n = 0
    for e in exprs:
        c = O.Cel(e)
        if c.rc == 1:
            continue
        m = CelModel(e)
        assert m.rc == c.rc, (e, m.rc, c.rc)
        if c.rc == 0:
            for r, md in zip(rows, models):
                assert m.eval(md, "aws", "r1", *r) == c.eval(md, "aws", "r1", *r), (e, r, md)
                n += 1
    assert n > 3000
    errs, rcs = collections.Counter(), collections.Counter()
    for e in cel_boundary_exprs() + cel_truth_exprs():
        c, m = O.Cel(e), CelModel(e)
        assert c.rc == m.rc, (e, c.rc, m.rc)
        rcs[m.rc] += 1
        if m.rc:
            continue   # an int result below zero in NewProgram's sanity evaluation (e.g. 1 - 2): refused at compile time
        got = m.eval("m", "b", "r", *MAXTOK)
        assert got == c.eval("m", "b", "r", *MAXTOK), (e, got)
        errs[got[0]] += 1
    assert all(errs[k] > 0 for k in range(6)) and rcs[2] < rcs[0] / 10, (errs, rcs)
