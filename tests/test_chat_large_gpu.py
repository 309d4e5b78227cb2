"""/v1/chat/completions passthroughs of any size through aigw_chat_translate_large_{host,device}: the translate pass's answers on
its own corpora, the oracle's bytes on long agent transcripts (test_chat_large_cpu.py), the scan's boundaries, every splice, the
limits, the device form's output space, other schemas and call composition."""
import json
import os

import numpy as np
import pytest

import _oracle as O
import _workload as W
import test_chat_large_cpu as L

pytestmark = pytest.mark.gpu

OK, E400, DECLINED = 0, 1, 4
R_TOO_LARGE, R_TOKENS, R_OPS, R_SCRATCH, R_OUT_SPACE, R_DEPTH, R_SCHEMA, R_ARENA = 1, 5, 6, 7, 8, 16, 19, 18
CAPACITY = (R_TOO_LARGE, R_TOKENS, R_OPS, R_SCRATCH, R_OUT_SPACE, R_ARENA)
VERSION = "2025-01-01-preview"
G = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.close()


def cfg(ctx, schema, override=None, cost=False, force=False):
    return ctx.cfg(schema, model_override=override, cost_configured=cost, force=force, api_version=VERSION if schema == "azure-openai" else None)


def run(ctx, fn, c, bodies):
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    res, out, _ = fn(c, arena, offs, lens)
    recs = ctx._records(bodies, res, out)
    for r, x in zip(recs, res):
        r["flags"] = int(x["flags"])
    return recs


def large(ctx, c, bodies):
    return run(ctx, ctx.chat_translate_large_host, c, bodies)


def small(ctx, c, bodies):
    return run(ctx, ctx.chat_translate_host, c, bodies)


KEYS = ("status", "path", "body", "body_kind", "model", "stream", "flags")


def same_as_translate_pass(bodies, got, ref, label):
    """equal to group 1, or declined; returns (compared, extra declines)"""
    compared = extra = 0
    for b, g, h in zip(bodies, got, ref):
        if h["status"] == DECLINED and h["reason"] in CAPACITY:
            continue
        if g["status"] == DECLINED and h["status"] != DECLINED:
            extra += 1
            continue
        assert all(g[k] == h[k] for k in KEYS), (label, b[:300], {k: (g[k], h[k]) for k in KEYS if g[k] != h[k]}, g["reason"], h["reason"])
        compared += 1
    return compared, extra


def _goldens():
    cases = json.load(open(os.path.join(G, "testupstream_cases.json"), encoding="utf-8"))["cases"]
    return [c["requestBody"].encode() for c in cases if c.get("path", "/v1/chat/completions") == "/v1/chat/completions" and "requestBody" in c]


ERRORS = [b'{"model": "something", "messages": [invalid json', b'{"model":"m","messages":[{"role":"wizard","content":"x"}]}',
          b'{"model":"m","messages":[{"content":"x"}]}', b'{"model":"m","messages":[{"role":"user","content":[{"text":"x"}]}]}',
          b'{"model":"m","messages":[{"role":"user","content":[{"type":"video","text":"x"}]}]}', b'{"model":"m","messages":[{"role":"assistant","content":5}]}',
          b'{"model":5,"messages":[]}', b'{"model":"m","messages":{}}', b'{"model":"m","temperature":"hot"}', b'{"model":"m","messages":[{"role":"system","content":null}]}',
          b'{"model":"m","thinking":{"type":"bogus"}}', b'{"model":"m","tool_choice":7}', b'{"model":"m","messages":[],"max_tokens":1.5}',
          b'{"model":"m","messages":[],"max_tokens":1.0}', b'{"model":"m","messages":[],"n":1e2}', b'{"model":"m","messages":[{"role":"user"}]}',
          b'{"model":"m","messages":[{"role":"user"},{"role":"user","content":7}]}',
          b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f","arguments":"not json"}}]}]}',
          b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f","arguments":"[1]"}}]}]}',
          b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f"}}]}]}',
          b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f","arguments":"{\\"a\\":1,\\"a\\":2}"}}]}]}',
          b'{"model":"m","messages":[{"role":"assistant","tool_calls":[{"id":"a","function":{"name":"f","arguments":"{\\"a\\":1.50}"}}]}]}',
          b'{"model":"m","tools":[{"type":"function","function":{"name":"f","parameters":{"b":1,"a":[1,2.0,{"c":null}]}}}]}',
          b'{"model":"m","tools":[{"type":"function","function":{"name":"f","parameters":{"b":1e5}}}]}']
EDGES = [b"", b" ", b"{}", b"null", b"[]", b'{"model":"m"}', b'{"messages":[]}', b'{"model":"m","messages":[]} trailing', b'\n {"model":"m"} \n',
         b'{"model":"m","model":"n"}', b'{"model":"m\\u0041"}', b'{"mod\\u0065l":"m"}', b'{"model":"m","messages":[{"role":"user","content":"\\ud83d\\ude00"}]}',
         b'{"model":"m","messages":[{"role":"user","content":"\\ud83d"}]}', b'{"model":"m","x":"\\ude00"}', b'{"stream":true}', b'  {"stream":true,"stream_options":null}\n',
         b'{"stream":true,"stream_options":{}}', b'{"stream":true,"stream_options":{"x":1}}', b'{"model":null,"stream":true,"stream_options":{"include_usage":null}}',
         b'{"messages":[],"stream":true,"stream_options":{"include_usage":true}}', b'{"stream":true,"stream_options":{"include_usage":false},"model":"q"}',
         b'{"model":"m","response_format":{"type":"json_object"}}', b'{"model":"m","stream":"yes"}', b'{"model":"m","messages":[{"role":"user","content":"a\x01b"}]}',
         b'{"model":"m","messages":[{"role":"user","content":"a\\qb"}]}', b'{"model":"m"', b'{"model":"m"}}', b'{"a":[1 2]}', b'{"a":01}']


def _translate_corpora():
    arena, offs, lens = W.chat_corpus(2, 5000, 1500)
    bench = [bytes(arena[int(offs[i]):int(offs[i]) + int(lens[i])]) for i in range(len(lens))]
    return {"goldens": _goldens(), "bench": bench, "diverse": [W.diverse_body(s) for s in range(1500)], "errors": ERRORS, "edges": EDGES}


CONFIGS = [(s, ov, cost, force) for s in ("openai", "azure-openai") for ov in (None, "override-model") for cost in (False, True) for force in (False, True)]


def test_translate_corpora(ctx):
    corpora = _translate_corpora()
    totals = {}
    for schema, ov, cost, force in CONFIGS:
        c = cfg(ctx, schema, ov, cost, force)
        for name, bodies in corpora.items():
            n, extra = same_as_translate_pass(bodies, large(ctx, c, bodies), small(ctx, c, bodies), (schema, ov, cost, force, name))
            t = totals.setdefault(name, [0, 0]); t[0] += n; t[1] += extra
    print("\ncompared with the translate pass (bodies, extra declines):", totals)
    assert totals["bench"][1] == 0 and totals["bench"][0] >= 1500 * len(CONFIGS)
    assert totals["goldens"][1] == 0


def check_oracle(schema, bodies, got, override=None, cost=False, force=False):
    for b, g in zip(bodies, got):
        t = O.chat_translate(schema, b, model_override=override or "", cost_configured=cost, force=force, prefix=VERSION if schema == "azure-openai" else "v1")
        assert g["status"] == OK and t.status == O.OK, (schema, len(b), g["status"], g["reason"], t.err)
        assert g["path"].decode() == t.path and g["body_kind"] == t.body_kind and g["model"] == t.model and g["stream"] == t.stream, (len(b), g["path"], t.path)
        assert g["body"] == (t.body if t.body_kind == O.BYTES else b""), (schema, len(b), len(g["body"]), len(t.body))


@pytest.mark.parametrize("schema,ov,cost,force", CONFIGS)
def test_large_realistic(ctx, schema, ov, cost, force):
    bodies = L.realistic_corpus()
    got = large(ctx, cfg(ctx, schema, ov, cost, force), bodies)
    check_oracle(schema, bodies, got, ov, cost, force)
    for b, g in zip(bodies, got):   # bit 1: include_usage forced on a stream that does not ask for it
        j = json.loads(b)
        forced = bool(cost and j.get("stream") and not ((j.get("stream_options") or {}).get("include_usage") is True))
        assert g["flags"] == (1 if j.get("stream") else 0) | (2 if forced else 0)


def test_large_errors_are_400(ctx):
    base = L.long_chat(3, 200 << 10, "true")
    bad = [base.replace(b'"role":"tool"', b'"role":"wizard"', 1), base.replace(b'"temperature":0.2', b'"temperature":"hot"', 1), base[:-1], base + b"x",
           base.replace(b'"max_completion_tokens":4096', b'"max_completion_tokens":1.5', 1)]
    for b in bad:
        assert O.chat_translate("openai", b).status == 1, b[-80:]
    for schema in ("openai", "azure-openai"):
        got = large(ctx, cfg(ctx, schema), bad)
        assert [g["status"] for g in got] == [E400] * len(bad), [(g["status"], g["reason"]) for g in got]


def test_boundaries(ctx):
    bodies = L.boundary_bodies()
    for schema, ov, cost, force in [("openai", "ovr", True, False), ("azure-openai", None, True, False), ("openai", None, False, True)]:
        c = cfg(ctx, schema, ov, cost, force)
        got = large(ctx, c, bodies)
        check_oracle(schema, bodies, got, ov, cost, force)
        short = [b for b in bodies if len(b) <= 65536]
        n, extra = same_as_translate_pass(short, large(ctx, c, short), small(ctx, c, short), "boundaries")
        assert extra == 0 and n == len(short)


def _splice_bodies():
    """edit A in each form (replace include_usage, append into stream_options, replace a null stream_options, append at the root)
    against edit B (replace the model, append at the root), both orders, with bytes outside the root braces"""
    big = b'"x":"' + b"p" * 70000 + b'"'
    out = []
    for so in (b'"stream_options":{"include_usage":false}', b'"stream_options":{"a":1}', b'"stream_options":{}', b'"stream_options":null', b""):
        for model in (b'"model":"m"', b'"model":null', b""):
            for order in (0, 1):
                parts = [p for p in ((so, model) if order == 0 else (model, so)) if p]
                members = b",".join([b'"stream":true'] + parts + [big])
                for ws in (b"", b"  \n"):
                    out.append(ws + b"{" + members + b"}" + ws)
    out.append(b' { } ')
    return out


@pytest.mark.parametrize("schema,ov,cost", [("openai", "ovr-1", True), ("openai", None, True), ("openai", "ovr-1", False), ("azure-openai", "dep", True)])
def test_splices(ctx, schema, ov, cost):
    bodies = _splice_bodies()
    check_oracle(schema, bodies, large(ctx, cfg(ctx, schema, ov, cost), bodies), ov, cost)


def test_limits(ctx):
    d48, d49 = L.limit_bodies()
    c = cfg(ctx, "openai", "o", True)
    g = large(ctx, c, [d48, d49])
    assert (g[0]["status"], g[1]["status"], g[1]["reason"]) == (OK, DECLINED, R_DEPTH)
    check_oracle("openai", [d48], g[:1], "o", True)
    assert small(ctx, c, [d49])[0]["reason"] == R_DEPTH
    big = L.near_16mib()
    g = large(ctx, c, [big, big + b" "])
    check_oracle("openai", [big], g[:1], "o", True)
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_TOO_LARGE)
    # a long tool-call arguments string declines (the serial bound)
    args = json.dumps({"content": "x" * (70 << 10)})
    b = json.dumps({"model": "m", "messages": [{"role": "assistant", "tool_calls": [{"id": "a", "function": {"name": "f", "arguments": args}}]}]}).encode()
    g = large(ctx, c, [b])[0]
    assert (g["status"], g["reason"]) == (DECLINED, R_SCRATCH)


def test_other_schemas_decline(ctx):
    bodies = [L.long_chat(5, 100 << 10), b'{"model":"m"}']
    for schema in ("aws-bedrock", "gcp-anthropicai", "gcp-vertexai", "emb-openai"):
        got = large(ctx, ctx.cfg(schema), bodies)
        assert all((g["status"], g["reason"]) == (DECLINED, R_SCHEMA) for g in got)


def test_device_out_space(ctx):
    import torch
    bodies = [L.long_chat(11, 300 << 10), L.long_chat(12, 90 << 10)]
    import aigw_b200 as A
    arena, offs, lens = A.pack_bodies(bodies)
    c = cfg(ctx, "openai", "ovr", True)
    d_b = torch.from_numpy(arena).cuda(); d_o = torch.from_numpy(offs.astype(np.uint64).view(np.int64)).cuda(); d_l = torch.from_numpy(lens.astype(np.uint32).view(np.int32)).cuda()
    for cap in (16, len(bodies[1]) + 4096):
        d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        d_r = torch.zeros(len(bodies) * 32, dtype=torch.uint8, device="cuda"); d_u = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.chat_translate_large_device(c, d_b.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), len(bodies), int(lens.max()), d_out.data_ptr(), cap, d_r.data_ptr(), d_u.data_ptr())
        res = d_r.cpu().numpy().view(A.DocResult)
        host = large(ctx, c, bodies)
        for i, x in enumerate(res):
            if int(x["status"]) == OK:
                assert int(x["body_len"]) == len(host[i]["body"])
            else:
                assert (int(x["status"]), int(x["reason"])) == (DECLINED, R_OUT_SPACE)
                assert int(x["body_len"]) == len(host[i]["path"]) + len(host[i]["body"])
        if cap == 16:
            assert all(int(x["status"]) == DECLINED for x in res)


def test_mixed_call(ctx):
    rng = np.random.default_rng(5)
    mixed = [L.long_chat(40 + i, int(rng.integers(1 << 10, 3 << 20)), L.STREAM_MODES[i % 9]) for i in range(10)] + [W.diverse_body(s) for s in range(50)] + EDGES
    c = cfg(ctx, "openai", "ovr", True)
    whole = large(ctx, c, mixed)
    order = list(rng.permutation(len(mixed)))
    rev = large(ctx, c, [mixed[i] for i in order])
    cut = len(mixed) // 3
    split = large(ctx, c, mixed[:cut]) + large(ctx, c, mixed[cut:])
    for i, j in enumerate(order):
        assert all(rev[i][k] == whole[j][k] for k in KEYS)
    for a, b in zip(whole, split):
        assert all(a[k] == b[k] for k in KEYS)
    assert sum(g["status"] == OK for g in whole[:10]) == 10


def test_token_capacity(ctx):
    """len / 2 + 1024 scan tokens fit; two more in a body of the same length decline with AIGW_R_TOKENS"""
    def body(k, length):
        s = b'{"model":"m","x":[' + b",".join([b"1"] * k) + b"]}"
        return s + b" " * (length - len(s))
    k = 3000
    length = 4 * k - 2024          # tokens 2k + 12 == length / 2 + 1024
    at, over = body(k, length), body(k + 1, length)
    assert len(at) == len(over) == length
    c = cfg(ctx, "openai", "o", True)
    g = large(ctx, c, [at, over])
    check_oracle("openai", [at], g[:1], "o", True)
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_TOKENS)


def test_arguments_total(ctx):
    """tool-call arguments are checked up to 256 KiB per request: four 60 KB strings pass, a fifth declines with AIGW_R_SCRATCH"""
    def body(n):
        calls = [{"id": "c%d" % i, "type": "function", "function": {"name": "f", "arguments": json.dumps({"content": "x" * 60000})}} for i in range(n)]
        return json.dumps({"model": "m", "messages": [{"role": "assistant", "tool_calls": calls}]}).encode()
    c = cfg(ctx, "openai", "o", True)
    g = large(ctx, c, [body(4), body(5)])
    check_oracle("openai", [body(4)], g[:1], "o", True)
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_SCRATCH)


def test_key_order_work_bound(ctx):
    """the key-order check of tool parameters is charged for the key bytes it compares: 64 long keys that differ only in their
    last byte decline with AIGW_R_SCRATCH, the same object with short keys passes"""
    def body(key_len):
        params = {"k" * (key_len - 2) + "%02d" % i: 1 for i in range(64)}
        return json.dumps({"model": "m", "messages": [], "tools": [{"type": "function", "function": {"name": "f", "parameters": params}}]}).encode()
    c = cfg(ctx, "openai", "o", True)
    g = large(ctx, c, [body(8), body(4096)])
    check_oracle("openai", [body(8)], g[:1], "o", True)
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_SCRATCH)
