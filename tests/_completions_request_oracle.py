"""CPU restatement of the /v1/completions request side (test infrastructure only).

  ParseBody: json.Unmarshal into openai.CompletionRequest       internal/endpointspec/endpointspec.go:203-212
  RequestBody: ":path" and the sjson model override             internal/translator/openai_completions.go:44-67
  openai.CompletionRequest, PromptUnion                         internal/apischema/openai/openai.go:1883-2010
  unmarshalJSONNestedUnion                                      internal/apischema/openai/union.go:18-67,161-185

The verdict is three-way, as in tests/_responses_request_oracle.py: OK (the reference decodes the body), FAIL (ParseBody's 400) or
OUT (in body order, before any failure, the body reaches something the library does not restate, so the GPU may DECLINE it).  The
members are walked in body order with the scanner primitives of tests/_responses_oracle.py.  OUT: an escaped member name, an
escaped model string, a repeated known member, "prompt":null (UnmarshalJSON is called with null; no fixture pins sonic there), a
float64 member, or a number anywhere in `stop` (interface{} decodes numbers as float64), with an exponent or more than 308
integer digits, a null root, and what the index stage declines (a raw control
character in a string, nesting deeper than 48).

The bytes of an accepted body come from the C++ oracle's sjson `set` restatement (oracle/translate.hpp, reached through the
body-mutation export), as for the /v1/responses request oracle.
"""
from _responses_oracle import FAIL, OK, OUT, _Fail, _number, _Out, _skip, _string, _ws
from _responses_request_oracle import MAX_DEPTH, _raw_limits

INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
F64_INT_DIGITS = 308   # no exponent and at most this many integer digits: below 1e308, so no float64 overflow
MEMBERS = dict(
    {k: "str" for k in ("model", "suffix", "user")}, **{k: "int" for k in ("best_of", "logprobs", "max_tokens", "n", "seed")},
    **{k: "f64" for k in ("frequency_penalty", "presence_penalty", "temperature", "top_p")}, echo="bool", stream="bool",
    prompt="prompt", logit_bias="bias", stop="any", stream_options="sopt")


def _int(p, i):
    """a Go int / int64: an integer literal within int64 → end"""
    c = p[i]
    if not (c == 0x2D or 0x30 <= c <= 0x39):
        raise _Fail
    j, is_int, _ = _number(p, i)
    if not is_int or not INT64_MIN <= int(p[i:j]) <= INT64_MAX:
        raise _Fail
    return j


def _f64(p, i):
    c = p[i]
    if not (c == 0x2D or 0x30 <= c <= 0x39):
        raise _Fail
    j, _, ie = _number(p, i)
    if b"e" in p[i:j] or b"E" in p[i:j] or ie - i - (c == 0x2D) > F64_INT_DIGITS:
        raise _Out
    return j


def _any(p, i):
    """interface{}: any JSON value, whose numbers decode as float64 (the float64 rule of _f64) → end"""
    j = _skip(p, i)
    k = i
    while k < j:
        c = p[k]
        if c == 0x22:
            k = _string(p, k)[0]
        elif c == 0x2D or 0x30 <= c <= 0x39:
            k = _f64(p, k)
        else:
            k += 1
    return j


def _bool(p, i):
    for w in (b"true", b"false"):
        if p.startswith(w, i):
            return i + len(w)
    raise _Fail


def _null(p, i):
    return p.startswith(b"null", i)


def _elements(p, i, elem):
    """the array at p[i] == '[': elem(p, j) → end for every element → end of the array"""
    i = _ws(p, i + 1)
    if i < len(p) and p[i] == 0x5D:
        return i + 1
    while True:
        i = _ws(p, elem(p, _ws(p, i)))
        if i >= len(p):
            raise _Fail
        if p[i] == 0x2C:
            i += 1
            continue
        if p[i] == 0x5D:
            return i + 1
        raise _Fail


def _members(p, i, member):
    """the object at p[i] == '{': member(key, j) → end for every member (an escaped name is OUT) → end of the object"""
    i = _ws(p, i + 1)
    if i < len(p) and p[i] == 0x7D:
        return i + 1
    while True:
        if i >= len(p) or p[i] != 0x22:
            raise _Fail
        j, key, esc = _string(p, i)
        if esc:
            raise _Out
        i = _ws(p, j)
        if i >= len(p) or p[i] != 0x3A:
            raise _Fail
        i = _ws(p, member(key.decode("latin-1"), _ws(p, i + 1)))
        if i >= len(p):
            raise _Fail
        if p[i] == 0x2C:
            i = _ws(p, i + 1)
            continue
        if p[i] == 0x7D:
            return i + 1
        raise _Fail


def _or_null(f):
    return lambda p, i: i + 4 if _null(p, i) else f(p, i)


def _prompt(p, i):
    """unmarshalJSONNestedUnion("prompt", …): the first element of an array picks []string, [][]int64 or []int64"""
    c = p[i]
    if c == 0x22:
        return _string(p, i)[0]
    if c == 0x6E:
        raise _Out
    if c != 0x5B:
        raise _Fail   # "invalid prompt type (must be string or array)"
    f = _ws(p, i + 1)
    if f >= len(p):
        raise _Fail
    if p[f] == 0x5D:
        return f + 1
    if p[f] == 0x22:
        return _elements(p, i, _or_null(lambda q, j: _string(q, j)[0] if q[j] == 0x22 else _fail()))
    if p[f] == 0x5B:
        return _elements(p, i, _or_null(lambda q, j: _elements(q, j, _or_null(_int)) if q[j] == 0x5B else _fail()))
    if p[f] == 0x2D or 0x30 <= p[f] <= 0x39:
        return _elements(p, i, _or_null(_int))
    raise _Fail       # "invalid prompt array element"


def _fail():
    raise _Fail


class _Request:
    def __init__(self, p):
        self.p = p
        self.model = b""
        self.stream = False
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
        if t == "any":
            return _any(p, i)
        if t == "prompt":
            return _prompt(p, i)
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
        if t == "bool":
            j = _bool(p, i)
            if key == "stream":
                self.stream = p[i] == 0x74
            return j
        if t == "int":
            return _int(p, i)
        if t == "f64":
            return _f64(p, i)
        if c != 0x7B:
            raise _Fail
        if t == "bias":   # map[string]int
            return _members(p, i, lambda k, j: j + 4 if _null(p, j) else _int(p, j))
        seen = set()      # *StreamOptions

        def opt(k, j):
            if k != "include_usage":
                return _skip(p, j)
            if k in seen:
                raise _Out
            seen.add(k)
            return j + 4 if _null(p, j) else _bool(p, j)
        return _members(p, i, opt)


def parse_body(body: bytes):
    """CompletionsEndpointSpec.ParseBody → (verdict, model bytes, stream)."""
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
        return FAIL, b"", False
    except _Out:
        v = OUT
    ctrl, depth = _raw_limits(body)
    if ctrl or depth > MAX_DEPTH:
        v = OUT
    return v, r.model, r.stream


def request_path(prefix="v1"):
    """path.Join("/", prefix, "completions")"""
    pfx = prefix.strip("/")
    return "/" + (pfx + "/" if pfx else "") + "completions"


def translate(body: bytes, model_override="", prefix="v1", force=False):
    """ParseBody + RequestBody → (verdict, path, body bytes or None for an unchanged body, model, stream)."""
    from _oracle import body_mutate
    v, model, stream = parse_body(body)
    if v != OK:
        return v, None, None, model, stream
    out = None
    if model_override:
        rc, out = body_mutate(body, [], [("model", '"%s"' % model_override)])
        assert rc == 0
    elif force:
        out = body
    return OK, request_path(prefix), out, model, stream
