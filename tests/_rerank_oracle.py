"""CPU restatement of Cohere /v2/rerank (test infrastructure only).

  ParseBody: json.Unmarshal into cohere.RerankV2Request          internal/endpointspec/endpointspec.go:364-373
  RequestBody: ":path" and the sjson model override              internal/translator/cohere_rerank_v2.go:40-66
  ResponseBody: json.NewDecoder into cohere.RerankV2Response     cohere_rerank_v2.go:73-108
  ResponseError: a non-JSON error body as RerankV2Error          cohere_rerank_v2.go:110-135
  the types                                                      internal/apischema/cohere/rerank_v2.go

Every decode gives one of three verdicts, as in the other request oracles: OK (the reference decodes the body), FAIL (its decode
error) or OUT (before any failure, in body order, the body reaches something the library does not restate, so the GPU may
DECLINE it).  Request side OUT: an escaped member name or model string, a repeated known member, a null root, and what the index
stage declines (a raw control character in a string, nesting deeper than 48).  Response side OUT: escaped or repeated known keys, a
float64 with an exponent or more than 308 integer digits, and a token count whose float64 lies outside (-1, 2^32), where Go's
uint32 conversion is implementation-defined.

The bytes of an accepted request come from the C++ oracle's sjson `set` restatement (oracle/translate.hpp, reached through the
body-mutation export), as for the other request oracles.
"""
from _completions_request_oracle import _elements, _fail, _int, _members, _null, _or_null
from _responses_oracle import FAIL, OK, OUT, _Fail, _number, _Out, _skip, _string, _Walk, _ws
from _responses_request_oracle import MAX_DEPTH, _raw_limits

F64_INT_DIGITS = 308
MEMBERS = {"model": "str", "query": "str", "documents": "docs", "top_n": "int", "max_tokens_per_doc": "int"}


# ================================================================ request
class _Request:
    def __init__(self, p):
        self.p = p
        self.model = b""
        self.seen = set()

    def member(self, key, i):
        p = self.p
        t = MEMBERS.get(key)
        if t is None:
            return _skip(p, i)
        if key in self.seen:
            raise _Out
        self.seen.add(key)
        if i >= len(p):
            raise _Fail
        if _null(p, i):
            return i + 4
        c = p[i]
        if t == "str":
            if c != 0x22:
                raise _Fail
            j, raw, esc = _string(p, i)
            if key == "model":
                if esc:
                    raise _Out
                self.model = raw
            return j
        if t == "int":
            return _int(p, i)
        if c != 0x5B:   # []string, null elements decode as ""
            raise _Fail
        return _elements(p, i, _or_null(lambda q, j: _string(q, j)[0] if q[j] == 0x22 else _fail()))


def parse_body(body: bytes):
    """RerankEndpointSpec.ParseBody → (verdict, model bytes)."""
    r = _Request(body)
    try:
        i = _ws(body, 0)
        if body.startswith(b"null", i):
            if _ws(body, i + 4) != len(body):
                raise _Fail
            raise _Out   # decodes to the zero request; the kernels decline a null root
        if _ws(body, _skip(body, i)) != len(body):   # a syntax error anywhere is the decoder's error, whatever precedes it
            raise _Fail
        if body[i] != 0x7B:
            raise _Fail
        _members(body, i, r.member)
        v = OK
    except _Fail:
        return FAIL, b""
    except _Out:
        v = OUT
    ctrl, depth = _raw_limits(body)
    if ctrl or depth > MAX_DEPTH:
        v = OUT
    return v, r.model


def request_path(version="v2"):
    """path.Join("/", version, "rerank"): path.Clean of the joined elements"""
    segs = []
    for s in version.split("/"):
        if s == "..":
            if segs:
                segs.pop()
        elif s not in ("", "."):
            segs.append(s)
    return "".join("/" + s for s in segs) + "/rerank"


def translate(body: bytes, model_override="", version="v2", force=False):
    """ParseBody + RequestBody → (verdict, path, body bytes or None for an unchanged body, model)."""
    from _oracle import body_mutate
    v, model = parse_body(body)
    if v != OK:
        return v, None, None, model
    out = None
    if model_override:
        rc, out = body_mutate(body, [], [("model", '"%s"' % model_override)])
        assert rc == 0
    elif force:
        out = body   # onRetry: the original bytes
    return OK, request_path(version), out, model


# ================================================================ response
F64 = "f64"
RESULT = ("obj", {"index": "int", "relevance_score": F64}, None)
META = ("obj", {
    "api_version": ("obj", {"version": "str", "is_deprecated": "bool", "is_experimental": "bool"}, None),
    "billed_units": ("obj", {k: F64 for k in ("images", "input_tokens", "output_tokens", "search_units", "classifications")}, None),
    "tokens": ("obj", {"input_tokens": (F64, "in"), "output_tokens": (F64, "out")}, "tokens"),
    "cached_tokens": F64, "warnings": ("arr", "str")}, None)
RESPONSE = ("obj", {"results": ("arr", RESULT), "id": "str", "meta": META}, None)


class _RerankWalk(_Walk):
    """_Walk with the float64 member: a number below the float64 overflow (no exponent, at most 308 integer digits restated);
    a named one is captured as uint32(float64(text))"""
    def value(self, i, t, depth):
        name = None
        if isinstance(t, tuple) and t[0] == F64:
            t, name = t
        if t != F64:
            return super().value(i, t, depth)
        p = self.p
        i = _ws(p, i)
        if i >= len(p):
            raise _Fail
        c = p[i]
        if c == 0x6E:
            if not p.startswith(b"null", i):
                raise _Fail
            return i + 4
        if not (c == 0x2D or 0x30 <= c <= 0x39):
            raise _Fail
        j, _, ie = _number(p, i)
        if b"e" in p[i:j] or b"E" in p[i:j] or ie - i - (c == 0x2D) > F64_INT_DIGITS:
            raise _Out
        if name:
            f = float(p[i:j])   # correctly rounded, as strconv.ParseFloat
            if not -1.0 < f < 4294967296.0:
                raise _Out
            self.caps[name] = int(f)   # truncation toward zero
        if j < len(p) and p[j] not in b" \t\n\r,}]":
            raise _Fail
        return j


def response_usage(body: bytes):
    """Buffered ResponseBody → (verdict, (input, output, total) with -1 for unset).  The response model is always the request's."""
    w = _RerankWalk(body)
    try:
        w.value(0, RESPONSE, 0)   # the first value counts, trailing bytes are ignored
        v = OK
    except _Fail:
        v = FAIL
    except _Out:
        v = OUT
    c = w.caps
    if v != OK:
        return v, None
    if not c.get("tokens"):
        return OK, (-1, -1, -1)
    inp, out = c.get("in"), c.get("out")
    return OK, (-1 if inp is None else inp, -1 if out is None else out, ((inp or 0) + (out or 0)) & 0xFFFFFFFF)


def _quote(b: bytes) -> bytes:
    """the raw body as a JSON string, as the library's other raw-body error messages (oracle/response_error.hpp, oj::enc_str)"""
    out = bytearray(b'"')
    for c in b:
        if c in (0x22, 0x5C):
            out += b"\\" + bytes([c])
        elif c in (0x0A, 0x0D, 0x09):
            out += {0x0A: b"\\n", 0x0D: b"\\r", 0x09: b"\\t"}[c]
        elif c < 0x20:
            out += b"\\u%04x" % c
        else:
            out.append(c)
    return bytes(out + b'"')


def response_error(body: bytes, non_json_content_type: bool):
    """ResponseError → (verdict, body or None when the upstream body is forwarded untouched).  OUT: bytes >= 0x80 (the library's
    raw-body quoting is ASCII only) and the empty body, which the reference answers with {"message":""}."""
    if not non_json_content_type:
        return OK, None
    if not body or any(c >= 0x80 for c in body):
        return OUT, b'{"message":""}' if not body else None
    return OK, b'{"message":' + _quote(body) + b"}"
