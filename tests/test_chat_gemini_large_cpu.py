"""Corpora of /v1/chat/completions requests for aigw_chat_gemini_translate_large_* (test_chat_gemini_large_gpu.py feeds them through
the GPU): long-context requests in the subset the Gemini plan accepts, with a large system instruction (a string, and text parts)
and developer turns between the others, long documents in multi-part user messages, runs of consecutive user messages (merged into
one content), assistant turns with text, refusal parts and no content, tools on both sides of the JSON-schema decision (subset
schemas under gemini-1.5 models, arbitrary schemas under gemini-2.5 / gemini-3), and every generation_config form.  Here: their
shape, that they are reproducible, the oracle's verdicts with and without an override, and the densest records."""
import json

import numpy as np
import pytest

import _oracle as O
import test_chat_large_cpu as L

SCHEMA = "gcp-vertexai"
MODELS = ["gemini-1.5-pro-002", "gemini-2.5-flash", "gemini-1.5-flash", "gemini-3-pro-preview"]
# flips the JSON-schema decision of the gemini-1.5 requests (their subset schemas then go out as parametersJsonSchema)
OVERRIDE = "gemini-2.5-pro-custom"
SIZES = (70_000, 130_000, 300_000, 1_000_000, 4_000_000)


def oracle(body, override=""):
    return O.chat_translate(SCHEMA, body, model_override=override)


def json_schema_side(model):
    """the Gemini plan's decision: parametersJsonSchema (any schema) rather than parameters (the re-marshal subset)"""
    return "gemini" in model and ("2.5" in model or "3" in model)


def subset_schema(rng, depth=0):
    """parameters inside the re-marshal subset: type, description, properties, items, required, enum"""
    props = {}
    for k in range(int(rng.integers(1, 5))):
        kind = int(rng.integers(4))
        if kind == 0 or depth >= 3:
            props["field_%d" % k] = {"type": "string", "description": L._text(rng, 40, escapes=False)}
        elif kind == 1:
            props["mode_%d" % k] = {"type": "string", "enum": ["fast", "slow", "auto"]}
        elif kind == 2:
            props["list_%d" % k] = {"type": "array", "items": subset_schema(rng, depth + 1)}
        else:
            props["obj_%d" % k] = subset_schema(rng, depth + 1)
    return {"type": "object", "description": "arguments", "properties": props, "required": sorted(props)[:1]}


def _gen_config(seed):
    """every generation_config form the plan emits, spread over the seeds"""
    forms = [{"n": 2, "seed": 0, "top_logprobs": 3, "logprobs": True},
             {"n": 0, "frequency_penalty": -0.25, "presence_penalty": 0.5, "logprobs": False},
             {"seed": 42, "stop": "END", "temperature": 0.123456},
             {"stop": ["END", "STOP"], "top_p": 0.95, "temperature": 1},
             {"stop": [], "top_logprobs": 0, "temperature": 0.7, "top_p": 1.5e-3}]
    g = dict(forms[seed % len(forms)])
    g["max_completion_tokens" if seed % 2 else "max_tokens"] = [8192, 0, 1024][seed % 3]
    return g


def gemini_chat(seed, target):
    """A long-context request of about `target` bytes in the Gemini plan's subset, serialised with ensure_ascii=False."""
    rng = np.random.default_rng(seed)
    model = MODELS[seed % len(MODELS)]
    big_sys = L._text(rng, max(2000, target // 20))
    if seed % 2:
        msgs = [{"role": "system", "content": big_sys}]
    else:
        msgs = [{"role": "system", "content": [{"type": "text", "text": big_sys[: len(big_sys) // 2]}, {"type": "text", "text": ""},
                                               {"type": "text", "text": big_sys[len(big_sys) // 2:]}]}]
    size = len(big_sys) + 500
    while size < target:
        r = rng.random()
        if r < 0.15:
            msgs.append({"role": "developer", "content": L._text(rng, 200)})
        elif r < 0.25:
            msgs.append({"role": "system", "content": [{"type": "text", "text": L._text(rng, 150)}]})
        # a long document in parts, or a run of short user messages that the plan merges into one content
        if rng.random() < 0.5:
            n = int(rng.integers(1000, max(2000, target // 8)))
            msgs.append({"role": "user", "content": [{"type": "text", "text": "Read this document:"}, {"type": "text", "text": L._text(rng, n)},
                                                     {"type": "text", "text": L._text(rng, 80)}]})
            size += n + 200
        else:
            for _ in range(int(rng.integers(1, 5))):
                n = int(rng.integers(20, 2000))
                msgs.append({"role": "user", "content": L._text(rng, n)})
                size += n + 40
        kind = rng.random()
        if kind < 0.4:
            msgs.append({"role": "assistant", "content": L._text(rng, int(rng.integers(50, 1500)))})
        elif kind < 0.7:
            msgs.append({"role": "assistant", "content": [{"type": "text", "text": L._text(rng, 300)}] + ([{"type": "refusal", "refusal": "no"}] if rng.random() < 0.3 else [])})
        elif kind < 0.8:
            msgs.append({"role": "assistant", "content": [{"type": "refusal", "refusal": "I can't"}]})
        elif kind < 0.9:
            msgs.append({"role": "assistant", "content": None})
        else:
            msgs.append({"role": "assistant", "content": "", "tool_calls": []})
        size += 800
    msgs.append({"role": "user", "content": "Summarise the above."})
    body = {"model": model, "messages": msgs}
    body.update(_gen_config(seed))
    ntools = int(rng.integers(0, 30)) if seed % 3 else 0
    tools = []
    for k in range(ntools):
        params = L._schema(rng) if json_schema_side(model) and rng.random() < 0.7 else subset_schema(rng)
        fn = {"name": "tool_%d" % k, "description": L._text(rng, 60, escapes=False), "parameters": params}
        if k % 7 == 3:
            fn["parameters"] = {}
        tools.append({"type": "function", "function": fn})
    if tools:
        body["tools"] = tools
    if seed % 2 == 0:
        body["stream"] = True
    return json.dumps(body, ensure_ascii=False).encode()


def gemini_corpus():
    return [gemini_chat(500 + i, t) for i, t in enumerate(SIZES)]


def subset_corpus():
    """the gemini-1.5 requests alone: their schemas are subset schemas, so the override flips their decision and they stay OK"""
    return [b for b in gemini_corpus() if not json_schema_side(json.loads(b)["model"])]


def small_corpus():
    """the generator's requests cut below 64 KiB, for the comparison with the translate pass"""
    return [gemini_chat(600 + i, t) for i, t in enumerate((3_000, 9_000, 25_000, 45_000))]


def escape_dense():
    """the corpus re-serialised with ensure_ascii: every non-ASCII character becomes a \\u escape in the text the plan copies
    (system text included), which it re-spells; the tool parameters hold none"""
    return [json.dumps(json.loads(b), ensure_ascii=True).encode() for b in gemini_corpus()[:3]]


def dense_shapes(n):
    """the densest records per body byte: a user text of \\b escapes (3.0x), alternating one-word user and assistant messages,
    and one-word user messages (merged into one content)"""
    b1 = b'{"model":"gemini-1.5-pro","messages":[{"role":"user","content":"' + b"\\b" * n + b'"}]}'
    b2 = json.dumps({"model": "gemini-1.5-pro", "messages": [{"role": "user", "content": "x"}, {"role": "assistant", "content": "x"}] * max(1, n // 66)},
                    separators=(",", ":")).encode()
    b3 = json.dumps({"model": "gemini-1.5-pro", "messages": [{"role": "user", "content": "x"}] * max(1, n // 30)}, separators=(",", ":")).encode()
    return [b1, b2, b3]


def test_corpus_shape_and_reproducible():
    # pinned: a change to the generators changes what the GPU tests compare, and shows here
    assert L.digest(gemini_corpus()) == DIGESTS["gemini"]
    assert L.digest(small_corpus()) == DIGESTS["small"]
    assert L.digest(escape_dense()) == DIGESTS["dense"]
    assert L.digest(dense_shapes(4000)) == DIGESTS["shapes"]
    sides = set()
    for b, t in zip(gemini_corpus(), SIZES):
        assert 0.9 * t < len(b) < 1.3 * t, (len(b), t)
        j = json.loads(b)
        roles = [m["role"] for m in j["messages"]]
        assert {"system", "user", "assistant"} <= set(roles) and "tool" not in roles
        assert roles[1:].count("system") + roles.count("developer") > 0
        assert any(roles[i] == roles[i + 1] == "user" for i in range(len(roles) - 1))
        assert any(m["role"] == "user" and isinstance(m["content"], list) and len(m["content"]) > 1 for m in j["messages"])
        asst = [m["content"] for m in j["messages"] if m["role"] == "assistant"]
        assert any(isinstance(c, list) for c in asst) and any(not c for c in asst)
        sides.add(json_schema_side(j["model"]))
    assert sides == {False, True}
    assert any("tools" in json.loads(b) for b in gemini_corpus())
    assert {k for b in gemini_corpus() + small_corpus() for k in json.loads(b)} >= {"n", "seed", "top_logprobs", "logprobs", "frequency_penalty",
                                                                                  "presence_penalty", "stop", "temperature", "top_p"}
    assert all(len(b) < 64 << 10 for b in small_corpus())
    assert all(b"\\u" in b for b in escape_dense())
    assert subset_corpus() and all(not json_schema_side(json.loads(b)["model"]) for b in subset_corpus())


@pytest.mark.parametrize("override", ["", OVERRIDE])
def test_oracle_accepts(override):
    bodies = gemini_corpus()[:4] + small_corpus() + escape_dense() if not override else subset_corpus() + small_corpus()
    for b in bodies:
        t = oracle(b, override)
        assert t.status == O.OK, (len(b), t.err)
        j = json.loads(t.body)
        assert set(j) <= {"contents", "tools", "generation_config", "system_instruction"}
        assert t.path.startswith("publishers/google/models/" + (override or json.loads(b)["model"]) + ":")
        assert t.stream == bool(json.loads(b).get("stream"))
        if "tools" in json.loads(b) and j["tools"]:
            decl = j["tools"][0]["functionDeclarations"]
            js = json_schema_side(override or json.loads(b)["model"])
            assert all(("parameters" not in d) or not js for d in decl) and all(("parametersJsonSchema" not in d) or js for d in decl)


def test_oracle_merges_users_and_keeps_system_last():
    b = gemini_corpus()[0]
    t = oracle(b)
    j = json.loads(t.body)
    roles = [c["role"] for c in j["contents"]]
    assert all(not (roles[i] == roles[i + 1] == "user") for i in range(len(roles) - 1))
    assert list(json.loads(t.body))[-1] == "system_instruction"


def test_oracle_record_ratios():
    """the densest shapes give the header's ratio; the host arena (3 * len per body) holds them"""
    b1, b2, b3 = dense_shapes(30000)
    r = [len(oracle(b).body) / len(b) for b in (b1, b2, b3)]
    assert 2.95 < r[0] < 3.01 and r[1] < 1.3 and r[2] < 0.5, r
    for b in (b1, b2, b3):
        assert len(oracle(b).path) + len(oracle(b).body) <= 3 * len(b) + 1024


DIGESTS = {"gemini": "e87df2428cde390653aa7824d41581170c40ace9d95cb3b0b1ddf3f1e796acce",
           "small": "c8a101168b5e1984b41bf6c82a3aa205b7ec1defc5a1de0464d644639ac12f34",
           "dense": "d5cf356f6c35a7b5e998984bd0547673ff82560de03bcd05fcf67f2b0b29265e",
           "shapes": "6551253123a19ada563b2f0f708077c51156e445cb75c1f7236b1717bce31059"}
