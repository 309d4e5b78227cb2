"""CPU restatement of the /v1/responses request side (test infrastructure only).

  ParseBody: json.Unmarshal into openai.ResponseRequest        internal/endpointspec/endpointspec.go:292-301
  RequestBody: ":path" and the sjson model override            internal/translator/openai_responses.go:50-78
  openai.ResponseRequest and its unions                        internal/apischema/openai/openai.go:2183-2400, 2415-2560,
                                                               2694-2792, 3477-4130, 4784-4820, 4977-5014, 5634-5720

The verdict is three-way, as in tests/_responses_oracle.py, whose walker this module extends: OK (the reference decodes the
body), FAIL (ParseBody's 400) or OUT (in body order, before any failure, the body reaches something the library's subset does
not restate, so the GPU may DECLINE it).  No failure is derived from a tag lookup: a tagged union whose tag the subset does not
restate, or that receives null or a non-object, is OUT.  The tag is taken as gjson takes it: the first top-level "type"; a
missing, null or empty tag is "".  An escaped member name anywhere in a union element, or an escaped tag or role, is OUT.

The bytes of an accepted body come from the C++ oracle's sjson `set` restatement (oracle/translate.hpp, reached through the
body-mutation export, whose JSON-value rule passes a quoted override through as the raw value), not from a second sjson here.
"""
from _responses_oracle import DECL, FAIL, OK, OUT, _Fail, _number, _Out, _skip, _string, _Walk, _ws

MAX_DEPTH = 48   # nesting the translate pass's grammar check accepts

RINT = ("rint",)                 # int64; more than 18 digits or "-0" is outside the subset (the kernels' integer rule)
OBJANY = ("objany",)             # map[string]any: an object (or null), contents unchecked
STRDECL = ("strdecl",)           # function_call_output.output: only the string form is restated
TEXTPART = ("obj", {"text": "str", "type": "str"}, None)
CONV = ("conv",)
TC = ("tc",)
IN_PARTS = {"input_text": TEXTPART,
            "input_image": ("obj", {"detail": "str", "file_id": "str", "image_url": "str", "type": "str"}, None),
            "input_file": ("obj", {"file_id": "str", "file_data": "str", "file_url": "str", "filename": "str", "type": "str"}, None)}
OUT_PARTS = {"output_text": ("obj", {"annotations": ("arr", DECL), "text": "str", "logprobs": ("arr", DECL), "type": "str"}, None),
             "refusal": ("obj", {"refusal": "str", "type": "str"}, None)}
EASY_CONTENT = ("strlist", IN_PARTS, True)      # (…, element tags, null decodes)
OUT_CONTENT = ("strlist", OUT_PARTS, False)
EASY = ("obj", {"content": EASY_CONTENT, "role": "str", "type": "str"}, None)
OUTMSG = ("obj", {"id": "str", "content": OUT_CONTENT, "status": "str", "role": "str", "type": "str"}, None)
ITEMS = {"function_call": ("obj", {k: "str" for k in ("arguments", "call_id", "name", "id", "status", "type")}, None),
         "function_call_output": ("obj", {"call_id": "str", "output": STRDECL, "id": "str", "status": "str", "type": "str"}, None),
         "reasoning": ("obj", {"id": "str", "summary": ("arr", TEXTPART), "encrypted_content": "str", "content": ("arr", TEXTPART),
                               "status": "str", "type": "str"}, None),
         "item_reference": ("obj", {"id": "str", "type": "str"}, None)}
INPUT = ("strlist", "items", True)
TOOLS = {"function": ("obj", {"strict": "bool", "parameters": OBJANY, "name": "str", "description": "str", "type": "str"}, None)}
TC_TAGS = {"function": ("obj", {"name": "str", "type": "str"}, None)}
FORMATS = {"text": ("obj", {"type": "str"}, None), "json_object": ("obj", {"type": "str"}, None),
           "json_schema": ("obj", {"name": "str", "schema": OBJANY, "strict": "bool", "description": "str", "type": "str"}, None)}
FORMAT = ("tagged", FORMATS)
REQUEST = ("obj", dict(
    {k: "bool" for k in ("background", "parallel_tool_calls", "store")},
    **{k: RINT for k in ("max_output_tokens", "max_tool_calls", "top_logprobs")},
    **{k: "str" for k in ("instructions", "previous_response_id", "prompt_cache_key", "safety_identifier", "user", "prompt_cache_retention",
                          "service_tier", "truncation")},
    stream=("bool", "stream"), temperature="float", top_p="float", presence_penalty="f32", frequency_penalty="f32", model=("str", "model"),
    include=("arr", "str"), metadata=("map", "str"), conversation=CONV, stream_options=("obj", {"include_obfuscation": "bool"}, None),
    reasoning=("obj", {"effort": "str", "generate_summary": "str", "summary": "str"}, None),
    text=("obj", {"verbosity": "str", "format": FORMAT}, None), tool_choice=TC, tools=("arr", ("tagged", TOOLS)), input=INPUT,
    prompt=DECL, context_management=DECL), None)


def _union_scan(p, i):
    """The object at p[i] == '{' → (tag, role, has_role, has_content): gjson's first top-level "type" (b"" when missing, null or
    empty) and "role".  An escaped member name, an escaped tag or role, or a tag of another JSON type is OUT."""
    tag = role = None
    has_role = has_content = False
    i = _ws(p, i + 1)
    while True:
        if i >= len(p):
            raise _Fail
        if p[i] == 0x7D:
            break
        if p[i] == 0x2C:
            i = _ws(p, i + 1)
        if i >= len(p) or p[i] != 0x22:
            raise _Fail
        j, key, esc = _string(p, i)
        if esc:
            raise _Out
        i = _ws(p, j)
        if i >= len(p) or p[i] != 0x3A:
            raise _Fail
        i = _ws(p, i + 1)
        if i >= len(p):
            raise _Fail
        if key == b"type" and tag is None:
            if p[i] == 0x22:
                _, tag, e = _string(p, i)
                if e:
                    raise _Out
            elif p.startswith(b"null", i):
                tag = b""
            else:
                raise _Out
        elif key == b"role" and not has_role:
            has_role = True
            if p[i] == 0x22:
                _, role, e = _string(p, i)
                if e:
                    raise _Out
        elif key == b"content":
            has_content = True
        i = _ws(p, _skip(p, i))
    return (tag or b""), role, has_role, has_content


class _RequestWalk(_Walk):
    def value(self, i, t, depth):
        p = self.p
        i = _ws(p, i)
        if i >= len(p):
            raise _Fail
        c = p[i]
        if t == ("bool", "stream"):
            self.caps["stream"] = p.startswith(b"true", i)
            return super().value(i, "bool", depth)
        if not (isinstance(t, tuple) and t[0] in ("rint", "objany", "strdecl", "conv", "tc", "tagged", "strlist")):
            return super().value(i, t, depth)
        kind = t[0]
        if kind == "rint":
            if c == 0x2D or 0x30 <= c <= 0x39:
                j, is_int, _ = _number(p, i)
                if is_int and (j - i - (c == 0x2D) > 18 or p[i:j] == b"-0"):
                    raise _Out
            return super().value(i, "int", depth)
        if kind == "objany":
            if c not in b"{n":
                raise _Fail
            return super().value(i, "any", depth)
        if kind == "strdecl":
            if c != 0x22:
                raise _Out
            return super().value(i, "str", depth)
        if kind in ("conv", "tc"):    # a string (null decodes as one), else {id} / the function tag
            if c in b'"n':
                return super().value(i, "str", depth)
            if c != 0x7B:
                if kind == "conv":
                    raise _Fail
                raise _Out   # tool_choice: "missing type field"
            return self.value(i, ("obj", {"id": "str"}, None) if kind == "conv" else ("tagged", TC_TAGS), depth)
        if kind == "tagged":
            if c != 0x7B:
                raise _Out
            tag = _union_scan(p, i)[0]
            v = t[1].get(tag.decode("latin-1"))
            if v is None:
                raise _Out
            return self.value(i, v, depth)
        # "strlist": a string, or a list of tagged elements
        if c == 0x22:
            return super().value(i, "str", depth)
        if c == 0x6E:
            if not t[2]:
                raise _Fail   # ResponseOutputMessageContentUnion.UnmarshalJSON("null") fails
            return super().value(i, "str", depth)
        if c != 0x5B:
            raise _Fail
        elem = ("item",) if t[1] == "items" else ("tagged", t[1])
        return super().value(i, ("arr", elem), depth) if elem[0] == "tagged" else self._items(i, depth)

    def _items(self, i, depth):
        p = self.p
        i = _ws(p, i + 1)
        if i < len(p) and p[i] == 0x5D:
            return i + 1
        while True:
            i = _ws(p, i)
            if i >= len(p):
                raise _Fail
            if p[i] != 0x7B:
                raise _Out   # no "type", no role: "cannot unmarshal unknown input type"
            tag, role, has_role, has_content = _union_scan(p, i)
            if tag == b"":
                if not (has_role and has_content):
                    raise _Out
                t = EASY
            elif tag == b"message":
                t = OUTMSG if role == b"assistant" else EASY   # a failed input-message decode falls back to the easy form
            elif tag.decode("latin-1") in ITEMS:
                t = ITEMS[tag.decode("latin-1")]
            else:
                raise _Out
            i = _ws(p, self.value(i, t, depth + 1))
            if i >= len(p):
                raise _Fail
            if p[i] == 0x2C:
                i += 1
                continue
            if p[i] == 0x5D:
                return i + 1
            raise _Fail


def _raw_limits(p):
    """(a raw control character inside a string, deepest nesting): what the translate pass's index stage declines"""
    depth = worst = 0
    ctrl = False
    i = 0
    while i < len(p):
        c = p[i]
        if c == 0x22:
            i += 1
            while i < len(p) and p[i] != 0x22:
                if p[i] < 0x20:
                    ctrl = True
                i += 2 if p[i] == 0x5C else 1
        elif c in b"{[":
            depth += 1
            worst = max(worst, depth)
        elif c in b"}]":
            depth -= 1
        i += 1
    return ctrl, worst


def parse_body(body: bytes):
    """ResponsesEndpointSpec.ParseBody → (verdict, model bytes, stream)."""
    w = _RequestWalk(body)
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
        e = w.value(0, REQUEST, 0)
        if _ws(body, e) != len(body):
            raise _Fail
        v = OK
    except _Fail:
        return FAIL, b"", False
    except _Out:
        v = OUT
    ctrl, depth = _raw_limits(body)
    if ctrl or depth > MAX_DEPTH:
        v = OUT
    return v, w.caps.get("model", b""), bool(w.caps.get("stream"))


def request_path(prefix="v1"):
    """path.Join("/", prefix, "responses")"""
    pfx = prefix.strip("/")
    return "/" + (pfx + "/" if pfx else "") + "responses"


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
