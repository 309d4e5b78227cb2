"""CPU restatement of the /v1/responses response side (test infrastructure only).

  ResponseBody, stream branch: handleStreamingResponse + extractUsageFromBufferEvent   internal/translator/openai_responses.go:102-192
  ResponseBody, buffered branch: handleNonStreamingResponse                           internal/translator/openai_responses.go:117-142
  openai.Response and its unions                                                      internal/apischema/openai/openai.go:5845-6039 …

Every decode returns a three-way verdict: OK (the reference decodes it), FAIL (the reference's decode fails: the stream skips
the line, the buffered call returns "failed to unmarshal body") or OUT (the input reaches, in document order before any failure,
something the library's subset does not restate: the GPU may DECLINE it).  The decode walks the bytes in document order, as
sonic does (CaseSensitive: true; control characters accepted in strings; UTF-8 not validated; escapes must be well-formed;
RFC 8259 numbers).  Where a null reaches a union's UnmarshalJSON, encoding/json's documented rule is restated: the method is
called with `null` (no fixture pins sonic's behaviour there).
"""

OK, FAIL, OUT = "ok", "fail", "out"
MAX_TYPED_DEPTH = 12   # nesting the typed walk restates; deeper objects are outside the subset


class _Fail(Exception):
    pass


class _Out(Exception):
    pass


WS = b" \t\n\r"


def _ws(p, i):
    while i < len(p) and p[i] in WS:
        i += 1
    return i


def _string(p, i):
    """p[i] == '"' → (end, raw contents, escaped)"""
    j = i + 1
    esc = False
    while j < len(p):
        c = p[j]
        if c == 0x22:
            return j + 1, p[i + 1:j], esc
        if c == 0x5C:
            esc = True
            if j + 1 >= len(p):
                raise _Fail
            e = p[j + 1]
            if e == 0x75:
                h = p[j + 2:j + 6]
                if len(h) < 4 or any(x not in b"0123456789abcdefABCDEF" for x in h):
                    raise _Fail
                j += 6
                continue
            if e not in b'"\\/bfnrt':
                raise _Fail
            j += 2
            continue
        j += 1
    raise _Fail


def _number(p, i):
    """→ (end, is_int, int_end)"""
    j = i
    if j < len(p) and p[j] == 0x2D:
        j += 1
    if j >= len(p):
        raise _Fail
    if p[j] == 0x30:
        j += 1
    elif 0x31 <= p[j] <= 0x39:
        while j < len(p) and 0x30 <= p[j] <= 0x39:
            j += 1
    else:
        raise _Fail
    int_end, is_int = j, True
    if j < len(p) and p[j] == 0x2E:
        is_int = False
        j += 1
        if j >= len(p) or not 0x30 <= p[j] <= 0x39:
            raise _Fail
        while j < len(p) and 0x30 <= p[j] <= 0x39:
            j += 1
    if j < len(p) and p[j] in b"eE":
        is_int = False
        j += 1
        if j < len(p) and p[j] in b"+-":
            j += 1
        if j >= len(p) or not 0x30 <= p[j] <= 0x39:
            raise _Fail
        while j < len(p) and 0x30 <= p[j] <= 0x39:
            j += 1
    return j, is_int, int_end


def _skip(p, i, depth=0):
    """any JSON value, syntax only → end"""
    i = _ws(p, i)
    if i >= len(p):
        raise _Fail
    c = p[i]
    if c == 0x22:
        return _string(p, i)[0]
    if c in b"{[":
        if depth >= 64:
            raise _Out   # the library's untyped skip holds 64 levels; the decoder accepts deeper values
        close = 0x7D if c == 0x7B else 0x5D
        i = _ws(p, i + 1)
        if i < len(p) and p[i] == close:
            return i + 1
        while True:
            if c == 0x7B:
                if i >= len(p) or p[i] != 0x22:
                    raise _Fail
                i = _ws(p, _string(p, i)[0])
                if i >= len(p) or p[i] != 0x3A:
                    raise _Fail
                i += 1
            i = _ws(p, _skip(p, i, depth + 1))
            if i >= len(p):
                raise _Fail
            if p[i] == 0x2C:
                i = _ws(p, i + 1)
                continue
            if p[i] == close:
                return i + 1
            raise _Fail
    for w in (b"true", b"false", b"null"):
        if p.startswith(w, i):
            return i + len(w)
    return _number(p, i)[0]


def _tag(p, i):
    """gjson.GetBytes(data, "type") on the object at p[i] == '{': the first top-level "type" member's string, or None when it is
    absent or not a string (no tag the unions know).  An escaped member name before it, or an escaped tag, is outside the subset."""
    i = _ws(p, i + 1)
    while True:
        if i >= len(p):
            raise _Fail
        if p[i] == 0x7D:
            return None
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
        if key == b"type":
            if i < len(p) and p[i] == 0x22:
                _, t, e = _string(p, i)
                if e:
                    raise _Out
                return t
            return None
        i = _ws(p, _skip(p, i))


# ---- the restated subset.  A type is: "str" | "int" | "float" | "f32" | "bool" | "any" | "created" | "pcreated" | "decline"
#      | ("obj", {key: type}, capture) | ("arr", elem) | ("map", elem) | ("union", {tag: type or "decline"}) | ("strobj", type)
#      | ("strarr", type).  Counters are captured by name.
DECL = "decline"
USAGE = ("obj", {"input_tokens": ("int", "in"), "input_tokens_details": ("obj", {"cached_tokens": ("int", "cached"), "cache_creation_input_tokens": ("int", "creation")}, None),
                 "output_tokens": ("int", "out"), "output_tokens_details": ("obj", {"reasoning_tokens": ("int", "reasoning")}, None), "total_tokens": ("int", "total")}, "usage")
TOPLP = ("obj", {"token": "str", "bytes": ("arr", "int"), "logprob": "float"}, None)
LOGPROB = ("obj", {"token": "str", "bytes": ("arr", "int"), "logprob": "float", "top_logprobs": ("arr", TOPLP)}, None)
ANNOT = ("union", {
    "file_citation": ("obj", {"file_id": "str", "filename": "str", "index": "int", "type": "str"}, None),
    "url_citation": ("obj", {"end_index": "int", "start_index": "int", "title": "str", "url": "str", "type": "str"}, None),
    "container_file_citation": ("obj", {"container_id": "str", "end_index": "int", "file_id": "str", "filename": "str", "start_index": "int", "type": "str"}, None),
    "file_path": ("obj", {"file_id": "str", "index": "int", "type": "str"}, None)})
PART = ("union", {"output_text": ("obj", {"annotations": ("arr", ANNOT), "text": "str", "logprobs": ("arr", LOGPROB), "type": "str"}, None),
                  "refusal": ("obj", {"refusal": "str", "type": "str"}, None)})
TEXTPART = ("obj", {"text": "str", "type": "str"}, None)
OUTPUT_TAGS = ["message", "file_search_call", "function_call", "function_call_output", "web_search_call", "computer_call", "reasoning", "compaction",
               "image_generation_call", "code_interpreter_call", "local_shell_call", "shell_call", "shell_call_output", "apply_patch_call",
               "apply_patch_call_output", "mcp_call", "mcp_list_tools", "mcp_approval_request", "custom_tool_call"]
ITEM = ("union", dict({t: DECL for t in OUTPUT_TAGS}, **{
    "message": ("obj", {"id": "str", "content": ("strarr", ("arr", PART)), "status": "str", "role": "str", "type": "str"}, None),
    "function_call": ("obj", {"arguments": "str", "call_id": "str", "name": "str", "id": "str", "status": "str", "type": "str"}, None),
    "reasoning": ("obj", {"id": "str", "summary": ("arr", TEXTPART), "encrypted_content": "str", "content": ("arr", TEXTPART), "status": "str", "type": "str"}, None)}))
TOOL_TAGS = ["function", "file_search", "computer_use_preview", "web_search", "web_search_2025_08_26", "mcp", "code_interpreter", "image_generation",
             "custom", "local_shell", "shell", "web_search_preview", "web_search_preview_2025_03_11", "apply_patch"]
TOOL = ("union", dict({t: DECL for t in TOOL_TAGS}, function=("obj", {"strict": "bool", "parameters": ("map", "any"), "name": "str", "description": "str", "type": "str"}, None)))
TOOL_CHOICE_TAGS = ["allowed_tools", "file_search", "web_search_preview", "computer_use_preview", "web_search_preview_2025_03_11", "image_generation",
                    "code_interpreter", "function", "mcp", "custom", "apply_patch", "shell"]
TOOL_CHOICE = ("strobj", ("union", dict({t: DECL for t in TOOL_CHOICE_TAGS}, function=("obj", {"name": "str", "type": "str"}, None))))
FORMAT = ("union", {"text": ("obj", {"type": "str"}, None), "json_object": ("obj", {"type": "str"}, None),
                    "json_schema": ("obj", {"name": "str", "schema": ("map", "any"), "strict": "bool", "description": "str", "type": "str"}, None)})
RESPONSE = ("obj", {
    "id": "str", "created_at": "created", "completed_at": "pcreated", "error": ("obj", {"code": "str", "message": "str"}, None),
    "incomplete_details": ("obj", {"reason": "str"}, None), "instructions": ("strobj", ("arr", DECL)), "metadata": ("map", "str"),
    "model": ("str", "model"), "object": "str", "output": ("arr", ITEM), "parallel_tool_calls": "bool", "temperature": "float",
    "tool_choice": TOOL_CHOICE, "tools": ("arr", TOOL), "top_p": "float", "background": "bool", "conversation": ("obj", {"id": "str"}, None),
    "max_output_tokens": "int", "max_tool_calls": "int", "previous_response_id": "str", "prompt": ("obj", {"id": "str", "variables": DECL, "version": "str"}, None),
    "prompt_cache_key": "str", "prompt_cache_retention": "str", "reasoning": ("obj", {"effort": "str", "generate_summary": "str", "summary": "str"}, None),
    "safety_identifier": "str", "service_tier": "str", "status": "str", "text": ("obj", {"format": FORMAT, "verbosity": "str"}, None),
    "top_logprobs": "int", "truncation": "str", "usage": USAGE, "user": "str", "presence_penalty": "f32", "frequency_penalty": "f32", "store": "bool"}, "response")
EVENT = ("obj", {"type": "str", "sequence_number": "int", "response": RESPONSE}, None)


class _Walk:
    def __init__(self, p):
        self.p = p
        self.caps = {}     # capture name → value (ints: low 32 bits; "model": bytes; objects: True)

    def value(self, i, t, depth):
        p = self.p
        i = _ws(p, i)
        if i >= len(p):
            raise _Fail
        c = p[i]
        name = None
        if isinstance(t, tuple) and t[0] in ("str", "int"):
            t, name = t
        if isinstance(t, tuple) and t[0] == "strobj":
            t = "str" if c in b'"n' else t[1]
        if isinstance(t, tuple) and t[0] == "strarr":   # a string, or the array; anything else (null included) is an error
            if c == 0x22:
                t = "str"
            elif c == 0x5B:
                t = t[1]
            else:
                raise _Fail
        if isinstance(t, tuple) and t[0] == "union":
            if c != 0x7B:
                raise _Fail   # null and non-objects have no "type"
            tag = _tag(p, i)
            v = t[1].get(tag.decode("latin-1")) if tag is not None else None
            if v is None:
                raise _Fail   # unknown tag
            t = v
        if t == DECL:
            raise _Out
        if t == "any":
            return _skip(p, i)
        if c == 0x6E:
            if not p.startswith(b"null", i):
                raise _Fail
            if t == "created":
                raise _Fail   # JSONUNIXTime.UnmarshalJSON("null") fails ParseInt
            return i + 4
        if t == "str":
            if c != 0x22:
                raise _Fail
            j, raw, esc = _string(p, i)
            if name == "model":
                if esc:
                    raise _Out
                self.caps["model"] = raw
            return j
        if t in ("int", "float", "f32", "created", "pcreated"):
            if not (c == 0x2D or 0x30 <= c <= 0x39):
                raise _Fail
            j, is_int, ie = _number(p, i)
            if j < len(p) and p[j] not in b" \t\n\r,}]":
                raise _Fail
            if t == "int":
                if not is_int:
                    raise _Fail
                v = int(p[i:j])
                if not -(1 << 63) <= v < (1 << 63):
                    raise _Fail
                if name:
                    self.caps[name] = v & 0xFFFFFFFF
            elif t == "f32":
                if b"e" in p[i:j] or b"E" in p[i:j] or ie - i - (c == 0x2D) > 38:
                    raise _Out   # float32 range is not restated
            elif t in ("created", "pcreated"):
                if not is_int and (ie >= j or p[ie] != 0x2E):
                    raise _Fail
                if not -(1 << 63) <= int(p[i:ie]) < (1 << 63):
                    raise _Fail
            return j
        if t == "bool":
            for w in (b"true", b"false"):
                if p.startswith(w, i):
                    return i + len(w)
            raise _Fail
        kind = t[0]
        if kind in ("obj", "map"):
            if c != 0x7B:
                raise _Fail
            if kind == "obj" and t[2]:
                self.caps[t[2]] = True
            i = _ws(p, i + 1)
            if i < len(p) and p[i] == 0x7D:
                return i + 1
            if depth >= MAX_TYPED_DEPTH:
                raise _Out
            seen = set()
            while True:
                if i >= len(p) or p[i] != 0x22:
                    raise _Fail
                j, key, esc = _string(p, i)
                if esc:
                    raise _Out
                i = _ws(p, j)
                if i >= len(p) or p[i] != 0x3A:
                    raise _Fail
                k = key.decode("latin-1")
                if kind == "map":
                    sub = t[1]
                else:
                    sub = t[1].get(k, "any")
                    if k in t[1]:
                        if k in seen:
                            raise _Out   # a repeated known member
                        seen.add(k)
                i = _ws(p, self.value(i + 1, sub, depth + 1))
                if i >= len(p):
                    raise _Fail
                if p[i] == 0x2C:
                    i = _ws(p, i + 1)
                    continue
                if p[i] == 0x7D:
                    return i + 1
                raise _Fail
        if kind == "arr":
            if c != 0x5B:
                raise _Fail
            i = _ws(p, i + 1)
            if i < len(p) and p[i] == 0x5D:
                return i + 1
            if depth >= MAX_TYPED_DEPTH:
                raise _Out
            while True:
                i = _ws(p, self.value(i, t[1], depth + 1))
                if i >= len(p):
                    raise _Fail
                if p[i] == 0x2C:
                    i += 1
                    continue
                if p[i] == 0x5D:
                    return i + 1
                raise _Fail
        raise AssertionError(t)


def _decode(p, t, trailing):
    w = _Walk(p)
    try:
        e = w.value(0, t, 0)
        if not trailing and _ws(p, e) != len(p):
            raise _Fail
    except _Fail:
        return FAIL, w.caps
    except _Out:
        return OUT, w.caps
    return OK, w.caps


class Usage:
    """metrics.TokenUsage: six counters and which of them are set (bit order of aigw_usage.mask)."""
    def __init__(self):
        self.input = self.output = self.total = self.cached = self.cache_creation = self.reasoning = 0
        self.mask = 0

    def set_all(self, c, creation):
        self.input, self.output, self.total = c.get("in", 0), c.get("out", 0), c.get("total", 0)
        self.cached, self.cache_creation, self.reasoning = c.get("cached", 0), creation, c.get("reasoning", 0)
        self.mask = 63

    def as_tuple(self):
        """(input, cached, cache_creation, output, total, reasoning), -1 for unset: the order of the library's stream results"""
        if self.mask != 63:
            return (-1,) * 6
        return (self.input, self.cached, self.cache_creation, self.output, self.total, self.reasoning)


def response_responses(body: bytes):
    """Buffered branch: json.NewDecoder(body).Decode(&openai.Response{}) (the first value counts, trailing bytes are ignored).
    → (verdict, Usage, model bytes).  model b"" means the caller falls back to the request model."""
    v, c = _decode(body, RESPONSE, trailing=True)
    u = Usage()
    if v != OK:
        return v, u, b""
    if c.get("usage"):
        u.set_all(c, c.get("creation", 0))
    return OK, u, c.get("model", b"")


class ResponsesSSEStream:
    """Stream branch.  No carry between calls: each call splits only its own bytes into lines."""
    def __init__(self, request_model=b""):
        self.request_model = request_model
        self.streaming_model = b""
        self.out = False   # an earlier call went outside the subset (the GPU may have declined the stream)

    def feed(self, chunk: bytes):
        """→ (verdict of the call, Usage).  OUT: some line of this call is outside the subset, or a response.completed event
        without usage (the reference dereferences a nil pointer and panics)."""
        u = Usage()
        verdict = OK
        for line in chunk.split(b"\n"):
            if not line.startswith(b"data: "):
                continue
            data = line[6:]
            if not data or data == b"[DONE]":
                continue
            try:
                i = _ws(data, 0)
                if i >= len(data) or data[i] != 0x7B:
                    continue
                tag = _tag(data, i)
            except _Fail:
                continue
            except _Out:
                verdict = OUT
                break
            if tag not in (b"response.created", b"response.completed"):
                continue   # every other event type changes nothing, whether or not it decodes
            v, c = _decode(data, EVENT, trailing=False)
            if v == FAIL:
                continue
            if v == OUT:
                verdict = OUT
                break
            if tag == b"response.created":
                if c.get("model"):
                    if len(c["model"]) > 160:
                        verdict = OUT
                        break
                    self.streaming_model = c["model"]
            else:
                if not c.get("response") or not c.get("usage"):
                    verdict = OUT
                    break
                u.set_all(c, 0)   # cache creation is always 0 on this path
        if verdict == OUT:
            self.out = True
        return verdict, u

    def model(self):
        return self.streaming_model or self.request_model
