"""Corpora of /v1/chat/completions requests for aigw_chat_bedrock_translate_large_* (test_chat_bedrock_large_gpu.py feeds them
through the GPU): test_chat_large_cpu's agent transcripts, and the shapes the AWS Bedrock Converse plan adds: system and developer
messages between other turns, long runs of tool messages crossing the scan's tiles, thinking / stop / service_tier, every
tool_choice form, models that need PathEscape, escape-dense transcripts, and the bodies whose record is densest.  Here: their
shape, that they are reproducible, and the oracle's verdicts."""
import json

import numpy as np
import pytest

import _oracle as O
import test_chat_large_cpu as L

TILE = L.TILE
TOOL_CHOICES = ["auto", "required", "none", {"type": "function", "function": {"name": "tool_0"}}, {"type": "function"}]


def bedrock_chat(seed, target, stream=True):
    """A transcript of about `target` bytes with the Converse plan's shapes: system / developer turns in the middle, runs of up to
    40 tool messages (some with text-part content), assistant text / refusal / thinking parts, thinking, stop, service_tier and a
    tool_choice form picked by the seed."""
    rng = np.random.default_rng(seed)
    tools = [{"type": "function", "function": {"name": "tool_%d" % k, "description": L._text(rng, 80), "parameters": L._schema(rng),
                                               **({"cache_control": {"type": "ephemeral"}} if k == 0 else {})}} for k in range(3)]
    msgs = [{"role": "system", "content": L._text(rng, 600)}]
    size, turn = 1000, 0
    while size < target:
        turn += 1
        r = rng.random()
        if r < 0.15:
            msgs.append({"role": "developer", "content": [{"type": "text", "text": L._text(rng, 300), "cache_control": {"type": "ephemeral"}}]})
        elif r < 0.25:
            msgs.append({"role": "system", "content": L._text(rng, 200)})
        msgs.append({"role": "user", "content": L._text(rng, int(rng.integers(50, 1500)))})
        parts = [{"type": "text", "text": L._text(rng, 100)}]
        if rng.random() < 0.3:
            parts.append({"type": "thinking", "text": L._text(rng, 200), "signature": "sig%d" % turn})
        if rng.random() < 0.1:
            parts.append({"type": "refusal", "refusal": "no"})
        ncalls = int(rng.integers(1, 40)) if rng.random() < 0.3 else int(rng.integers(1, 4))
        calls = [{"id": "c%d_%d" % (turn, c), "type": "function",
                  "function": {"name": "tool_%d" % (c % 3), "arguments": json.dumps({"q": L._text(rng, 30, escapes=False), "n": c, "deep": {"b": [1, 2], "a": None}})}}
                 for c in range(ncalls)]
        msgs.append({"role": "assistant", "content": parts, "tool_calls": calls})
        for c in calls:
            n = int(rng.integers(20, max(40, target // 200)))
            content = L._text(rng, n) if rng.random() < 0.7 else [{"type": "text", "text": L._text(rng, n)}]
            msgs.append({"role": "tool", "tool_call_id": c["id"], "content": content})
            size += n + 120
        size += 800
    body = {"model": ["anthropic.claude-3-5-sonnet", "us.amazon.nova-pro-v1:0", "arn:aws:bedrock:us-east-1:1:inference-profile/x y"][seed % 3],
            "messages": msgs, "tools": tools, "tool_choice": TOOL_CHOICES[seed % len(TOOL_CHOICES)], "temperature": 0.5, "top_p": 0.9,
            "max_tokens": 2048, "stop": ["END", "STOP"] if seed % 2 else "END"}
    if seed % 4 == 1:
        body["thinking"] = {"type": "enabled", "budget_tokens": 1024}
    elif seed % 4 == 2:
        body["thinking"] = {"type": "disabled"}
    if seed % 3 == 0:
        body["service_tier"] = "priority"
    if stream:
        body["stream"] = True
    return json.dumps(body).encode()


def bedrock_corpus():
    return [bedrock_chat(300 + i, t) for i, t in enumerate((70 << 10, 130 << 10, 300 << 10, 1 << 20))]


def escape_dense():
    """the realistic transcripts re-serialised with ensure_ascii: every non-ASCII character becomes a \\u escape"""
    return [json.dumps(json.loads(b), ensure_ascii=True).encode() for b in L.realistic_corpus(6, 64 << 10, 1 << 20)]


def tool_run_across_tiles():
    """one run of tool messages whose messages straddle the scan's 8 KiB tiles"""
    out = []
    for k in (200, 3000):
        msgs = [{"role": "user", "content": "go"}, {"role": "assistant", "tool_calls": [{"id": "a", "function": {"name": "f", "arguments": "{}"}}]}]
        msgs += [{"role": "tool", "tool_call_id": "t%d" % i, "content": "r" * (i % 97)} for i in range(k)]
        msgs.append({"role": "system", "content": "between"})
        msgs += [{"role": "tool", "tool_call_id": "u", "content": ""}, {"role": "user", "content": "end"}]
        out.append(json.dumps({"model": "m", "messages": msgs}).encode())
    return out


def dense_shapes(n):
    """the densest records per body byte: a string of \\b escapes (3x), empty tool messages (2.4x), and arguments holding a run
    of escaped backslashes, which shrink (each is spelled twice in the body, once in the record)"""
    b1 = b'{"model":"m","messages":[{"role":"user","content":"' + b"\\b" * n + b'"}]}'
    b2 = json.dumps({"model": "m", "messages": [{"role": "tool", "content": ""}] * max(1, n // 28)}, separators=(",", ":")).encode()
    b3 = json.dumps({"model": "m", "messages": [{"role": "assistant", "tool_calls": [{"id": "a", "function": {"name": "f", "arguments": json.dumps({"k": "\\" * min(n, 15000)})}}]}]}).encode()
    return [b1, b2, b3]


def path_models():
    """models that PathEscape keeps, escapes, and a ":path" at and above 65535 bytes"""
    base = {"messages": [{"role": "user", "content": "hi"}]}
    out = []
    for m in ("plain.model-1:0", "arn:aws:bedrock:us-east-1:1/x y", "café model%?#"):
        out.append(json.dumps(dict(base, model=m), ensure_ascii=False).encode())
    fixed = len("/model//converse")
    for k in ((65535 - fixed) // 3, (65535 - fixed) // 3 + 1):   # every byte escaped to three
        out.append(json.dumps(dict(base, model="/" * k)).encode())
    return out


def edge_requests():
    return [b'{"model":"m","stop":"x","messages":[{"role":"user","content":null}]}',
            b'{"model":"m","stop":[],"service_tier":"","messages":[{"role":"user","content":[{"type":"text","text":"a","cache_control":{"type":"ephemeral"}}]}]}',
            b'{"model":"anthropic.claude-v2","tool_choice":"my_tool","tools":[{"type":"function","function":{"name":"my_tool"}}],"messages":[]}',
            b'{"model":"nova","tool_choice":"my_tool","tools":[{"type":"function","function":{"name":"my_tool"}}],"messages":[]}',
            b'{"model":"m","tool_choice":{"type":"function","function":{"name":"f"}},"tools":[],"messages":[]}',
            b'{"model":"m","thinking":{"type":"enabled"},"messages":[{"role":"assistant","content":{"type":"thinking","text":"t","signature":""}}]}',
            b'{"model":"m","thinking":{"type":"adaptive"},"messages":[{"role":"assistant","content":""},{"role":"tool","content":[]}]}',
            b'{"model":"m","messages":[{"role":"system","content":[]},{"role":"developer","content":"d"}]}',
            b'{"model":"m","messages":[{"role":"user","content":"a\\/b\\u00e9\\ud83d\\ude00\\u0001\\f"}]}']


def test_corpus_shape_and_reproducible():
    # pinned: a change to the generators changes what the GPU tests compare, and shows here
    assert L.digest(bedrock_corpus()) == DIGESTS["bedrock"]
    assert L.digest(escape_dense()) == DIGESTS["dense"]
    assert L.digest(tool_run_across_tiles() + dense_shapes(4000) + path_models() + edge_requests()) == DIGESTS["shapes"]
    for b in bedrock_corpus():
        j = json.loads(b)
        roles = [m["role"] for m in j["messages"]]
        assert {"system", "user", "assistant", "tool"} <= set(roles)
        assert any(roles[i] == roles[i + 1] == "tool" for i in range(len(roles) - 1))
    assert all(b"\\u" in b for b in escape_dense())
    assert all(len(b) > 3 * TILE for b in tool_run_across_tiles()[1:])


@pytest.mark.parametrize("override", ["", "us.anthropic.claude-3-7 sonnet"])
def test_oracle_accepts(override):
    for b in bedrock_corpus() + escape_dense() + tool_run_across_tiles() + dense_shapes(20000) + path_models()[:3]:
        t = O.chat_translate("aws-bedrock", b, model_override=override)
        assert t.status == O.OK, (len(b), t.err)
        assert t.path.startswith("/model/") and json.loads(t.body)


def arguments_body(args: bytes) -> bytes:
    """one tool call whose "arguments" string holds the raw bytes `args` (quotes, backslashes and newlines escaped once)"""
    esc = args.replace(b"\\", b"\\\\").replace(b'"', b'\\"').replace(b"\n", b"\\n")
    return b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f","arguments":"' + esc + b'"}}]}]}'


# arguments texts with non-ASCII content: U+2028, invalid UTF-8 (0xFF 0xFE), a raw UTF-8-encoded surrogate, and whitespace, an
# exponent and escapes the re-serialisation drops or keeps
NONASCII_ARGS = [b'{"s":" \xe2\x80\xa8 \xc3\xa9"}', b'{"s":"\xff\xfe"}', b'{"s":"\xed\xa0\x80"}',
                 b'{"a" : [1, 2.5e3, true] , "b":{"y":null,"x":"\\n\\"q\\""}}']


def tool_use_input(record_body: bytes) -> bytes:
    """the bytes of the record's first toolUse input"""
    i = record_body.index(b'"input":') + len(b'"input":')
    return record_body[i:record_body.index(b',"toolUseId":', i)]


def test_oracle_record_ratios():
    """the densest shapes give the header's ratios; the oracle re-serialises arguments to no more bytes than their unescaped
    text, non-ASCII and invalid UTF-8 included (the scratch for re-serialised arguments is sized on that)"""
    b1, b2, b3 = dense_shapes(30000)
    r = [len(O.chat_translate("aws-bedrock", b).body) / len(b) for b in (b1, b2, b3)]
    assert 2.9 < r[0] < 3.01 and 2.3 < r[1] < 2.5 and r[2] < 1, r
    for args in NONASCII_ARGS:
        t = O.chat_translate("aws-bedrock", arguments_body(args))
        assert t.status == O.OK, (args, t.err)
        inp = tool_use_input(t.body)
        assert len(inp) <= len(args), (args, inp)
        if args[:4] == b'{"s"':
            assert inp == args   # compact already: the non-ASCII bytes are kept as they are


DIGESTS = {"bedrock": "66cd970c8292e53b0e9421ef9a5ff11d89d43edc44610505ffdf2a5536ec597d",
           "dense": "00a9ea26ab7181c4e581e2edeed2593243e49d899f866c79830e2f93bfbf029a",
           "shapes": "e6b84adcdb3e521446971df89ea283ade782ef9a1c6406ef9fab6ef746a304a9"}
