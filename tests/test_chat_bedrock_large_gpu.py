"""/v1/chat/completions to AWS Bedrock Converse at any size through aigw_chat_bedrock_translate_large_{host,device}: the translate
pass's answers (group 0) on its own corpora, the oracle's bytes above 64 KiB (test_chat_bedrock_large_cpu.py's corpora and
test_chat_large_cpu's transcripts), 400s / 422s / 500s deep in a body, the scan's boundaries, the limits, one-byte mutations, the
device form's output space, call composition and other schemas."""
import json

import numpy as np
import pytest

import _oracle as O
import test_chat_bedrock_large_cpu as B
import test_chat_large_cpu as L
import test_chat_large_gpu as G

pytestmark = pytest.mark.gpu

OK, E400, E422, INTERNAL, DECLINED = 0, 1, 2, 3, 4
R_TOO_LARGE, R_TOKENS, R_OPS, R_SCRATCH, R_OUT_SPACE, R_DEPTH, R_SCHEMA = 1, 5, 6, 7, 8, 16, 19
KEYS = ("status", "path", "body", "body_kind", "model", "stream", "flags")
ctx = G.ctx


def cfg(ctx, override=None):
    return ctx.cfg("aws-bedrock", model_override=override)


def large(ctx, c, bodies):
    return G.run(ctx, ctx.chat_bedrock_translate_large_host, c, bodies)


def check_oracle(bodies, got, override=None):
    for b, g in zip(bodies, got):
        t = O.chat_translate("aws-bedrock", b, model_override=override or "")
        assert g["status"] == t.status, (len(b), g["status"], g["reason"], t.status, t.err)
        if t.status == O.OK:
            assert g["path"].decode() == t.path and g["model"] == t.model and g["stream"] == t.stream, (len(b), g["path"][:80], t.path[:80])
            assert g["body"] == t.body, (len(b), len(g["body"]), len(t.body))


def test_translate_corpora(ctx):
    corpora = G._translate_corpora()
    corpora["shapes"] = [b for b in B.tool_run_across_tiles()[:1] + B.path_models()[:3] + B.edge_requests() if len(b) <= 65536]
    totals = {}
    for ov in (None, "us.anthropic.claude-3-7-sonnet"):
        c = cfg(ctx, ov)
        for name, bodies in corpora.items():
            n, extra = G.same_as_translate_pass(bodies, large(ctx, c, bodies), G.small(ctx, c, bodies), (ov, name))
            t = totals.setdefault(name, [0, 0]); t[0] += n; t[1] += extra
    print("\ncompared with the translate pass (bodies, extra declines):", totals)
    assert totals["bench"][1] == 0 and totals["bench"][0] >= 1500 * 2
    assert totals["goldens"][1] == 0


@pytest.mark.parametrize("ov", [None, "us.anthropic.claude-3-7 sonnet"])
def test_large_realistic(ctx, ov):
    bodies = L.realistic_corpus() + B.bedrock_corpus() + B.escape_dense()
    got = large(ctx, cfg(ctx, ov), bodies)
    assert all(g["status"] == OK for g in got), [(i, g["status"], g["reason"]) for i, g in enumerate(got) if g["status"] != OK]
    check_oracle(bodies, got, ov)
    for b, g in zip(bodies, got):
        assert g["flags"] == (1 if json.loads(b).get("stream") else 0) and g["body_kind"] == O.BYTES


def test_shapes(ctx):
    bodies = B.tool_run_across_tiles() + B.dense_shapes(20000) + B.path_models() + B.edge_requests()
    got = large(ctx, cfg(ctx), bodies)
    n = len(B.tool_run_across_tiles()) + 3
    check_oracle(bodies[:n + 4], got[:n + 4])
    assert (got[n + 4]["status"], got[n + 4]["reason"]) == (DECLINED, R_TOO_LARGE)   # a ":path" of 65536 bytes
    check_oracle(bodies[n + 5:], got[n + 5:])


def test_errors_deep(ctx):
    base = L.long_chat(3, 1 << 20, "true")
    bad400 = [base.replace(b'"role":"tool"', b'"role":"wizard"', 1), base.replace(b'"temperature":0.2', b'"temperature":"hot"', 1), base[:-1]]
    i = base.rindex(b'{"role":"tool"')
    no_content = base[:i] + b'{"role":"user"},' + base[i:]
    j = base.rindex(b'"arguments":"')
    not_json = base[:j] + b'"arguments":"not json' + base[j + len(b'"arguments":"'):]
    bodies = bad400 + [no_content, not_json]
    got = large(ctx, cfg(ctx), bodies)
    assert [g["status"] for g in got] == [E400, E400, E400, E422, INTERNAL], [(g["status"], g["reason"]) for g in got]
    check_oracle(bodies, got)


def test_boundaries(ctx):
    bodies = L.boundary_bodies()
    c = cfg(ctx, "ovr")
    got = large(ctx, c, bodies)
    check_oracle(bodies, got, "ovr")
    short = [b for b in bodies if len(b) <= 65536]
    n, extra = G.same_as_translate_pass(short, large(ctx, c, short), G.small(ctx, c, short), "boundaries")
    assert extra == 0 and n == len(short)


def test_limits(ctx):
    c = cfg(ctx)
    d48, d49 = L.limit_bodies()
    big = L.near_16mib()
    g = large(ctx, c, [d48, d49, big, big + b" "])
    assert (g[1]["status"], g[1]["reason"], g[3]["status"], g[3]["reason"]) == (DECLINED, R_DEPTH, DECLINED, R_TOO_LARGE)
    check_oracle([d48, big], [g[0], g[2]])


def _calls_body(raw_lens):
    """tool calls whose "arguments" strings are raw_lens[i] bytes long in the body: {"c":"xxx"} (12 bytes of envelope once escaped),
    or {} for a length of 2"""
    calls = [{"id": "c%d" % i, "type": "function", "function": {"name": "f", "arguments": "{}" if n == 2 else '{"c":"' + "x" * (n - 12) + '"}'}}
             for i, n in enumerate(raw_lens)]
    return json.dumps({"model": "m", "messages": [{"role": "assistant", "tool_calls": calls}]}).encode()


def test_arguments_edges(ctx):
    """an "arguments" string of 64 KiB translates and one byte more declines; so do 256 KiB of them in a request and one byte more
    (AIGW_R_SCRATCH, the serial bound of the walk)"""
    under = [_calls_body([65536]), _calls_body([65536, 65536, 65536, 65534, 2])]
    over = [_calls_body([65537]), _calls_body([65536, 65536, 65536, 65535, 2])]
    for b in under + over:
        j = json.loads(b)["messages"][0]["tool_calls"]
        assert sum(len(json.dumps(c["function"]["arguments"])) - 2 for c in j) in (65536, 65537, 262144, 262145)
    g = large(ctx, cfg(ctx), under + over)
    check_oracle(under, g[:2])
    assert [(x["status"], x["reason"]) for x in g[2:]] == [(DECLINED, R_SCRATCH)] * 2


ANY_WORK = 1 << 18


def _cmp_keys(a, b):
    m = min(len(a), len(b))
    k = 0
    while k < m and a[k] == b[k]:
        k += 1
    return (-1 if a[k] < b[k] else 1) if k < m else (0 if len(a) == len(b) else (-1 if len(a) < len(b) else 1)), k + 1


def any_work(keys):
    """the key-order check's work over one flat object as emit_any charges it (one unit per member visit, k + 1 per compare that
    reads k equal bytes, checked at each visit): the total, or None when it passes the budget"""
    work, last = 0, None
    while True:
        best = None
        for i, m in enumerate(keys):
            work += 1
            if work > ANY_WORK:
                return None
            c1 = 1
            if last is not None:
                c1, w = _cmp_keys(m, keys[last]); work += w
            if c1 > 0:
                if best is None:
                    best = i
                else:
                    c2, w = _cmp_keys(m, keys[best]); work += w
                    if c2 < 0:
                        best = i
        if best is None:
            return work
        last = best


def test_key_order_budget_edge(ctx):
    """64 parameter keys that differ in their last two bytes: the longest key length within the 2^18 units of work translates, one
    byte longer declines with AIGW_R_SCRATCH"""
    def keys(n):
        return ["k" * (n - 2) + "%02d" % i for i in range(64)]
    n = max(k for k in range(3, 200) if any_work([x.encode() for x in keys(k)]) is not None)
    assert n == 43 and any_work([x.encode() for x in keys(n + 1)]) is None

    def body(k):
        params = {x: 1 for x in keys(k)}
        return json.dumps({"model": "m", "messages": [], "tools": [{"type": "function", "function": {"name": "f", "parameters": params}}]}).encode()
    g = large(ctx, cfg(ctx), [body(n), body(n + 1)])
    check_oracle([body(n)], g[:1])
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_SCRATCH)


def test_op_capacity(ctx):
    """len / 2 + 4096 copy ops: a user string of "\\/a" repeated k times costs two ops per three bytes (a scratch op for each
    re-spelled slash, a body op for each "a" between them), and the record 2k + 10 in all.  The last k within the cap translates
    as the oracle does; one more declines with AIGW_R_OPS"""
    def body(k):
        return b'{"model":"m","messages":[{"role":"user","content":"' + b"\\/a" * k + b'"}]}'

    def fits(k):
        return 2 * k + 10 <= len(body(k)) // 2 + 4096
    k = max(x for x in range(1, 20000) if fits(x))
    assert k == 8227 and not fits(k + 1)
    g = large(ctx, cfg(ctx), [body(k), body(k + 1)])
    check_oracle([body(k)], g[:1])
    assert (g[1]["status"], g[1]["reason"]) == (DECLINED, R_OPS)
    assert O.chat_translate("aws-bedrock", body(k + 1)).status == O.OK


def test_arguments_bytes(ctx):
    """tool-call arguments with U+2028, invalid UTF-8 and a raw surrogate are re-serialised byte for byte as the oracle does"""
    bodies = [B.arguments_body(a) for a in B.NONASCII_ARGS]
    g = large(ctx, cfg(ctx), bodies)
    assert all(x["status"] == OK for x in g[:3]), [(x["status"], x["reason"]) for x in g]
    check_oracle(bodies[:3], g[:3])
    if g[3]["status"] == OK:   # 2.5e3 is not canonical: the translate pass declines it (AIGW_R_NUMBER) rather than reprint it
        check_oracle(bodies[3:], g[3:])


def test_other_schemas_decline(ctx):
    bodies = [L.long_chat(5, 100 << 10), b'{"model":"m"}']
    for schema in ("openai", "azure-openai", "gcp-anthropicai", "gcp-vertexai"):
        got = large(ctx, ctx.cfg(schema), bodies)
        assert all((g["status"], g["reason"]) == (DECLINED, R_SCHEMA) for g in got)
    # and the passthrough call keeps declining Bedrock
    got = G.large(ctx, cfg(ctx), bodies)
    assert all((g["status"], g["reason"]) == (DECLINED, R_SCHEMA) for g in got)


def test_device_out_space(ctx):
    import torch
    import aigw_b200 as A
    bodies = [L.long_chat(11, 300 << 10)] + B.dense_shapes(30000)[:2]
    arena, offs, lens = A.pack_bodies(bodies)
    c = cfg(ctx)
    host = large(ctx, c, bodies)   # the host form retries what did not fit its first arena: every record is whole
    check_oracle(bodies, host)
    d_b = torch.from_numpy(arena).cuda(); d_o = torch.from_numpy(offs.astype(np.uint64).view(np.int64)).cuda(); d_l = torch.from_numpy(lens.astype(np.uint32).view(np.int32)).cuda()
    for cap in (16, len(bodies[1]) * 3 + 4096):
        d_out = torch.zeros(cap + 64, dtype=torch.uint8, device="cuda")
        d_r = torch.zeros(len(bodies) * 32, dtype=torch.uint8, device="cuda"); d_u = torch.zeros(1, dtype=torch.int64, device="cuda")
        ctx.chat_bedrock_translate_large_device(c, d_b.data_ptr(), d_o.data_ptr(), d_l.data_ptr(), len(bodies), int(lens.max()), d_out.data_ptr(), cap, d_r.data_ptr(), d_u.data_ptr())
        res = d_r.cpu().numpy().view(A.DocResult)
        for i, x in enumerate(res):
            if int(x["status"]) == OK:
                assert int(x["body_len"]) == len(host[i]["body"])
            else:
                assert (int(x["status"]), int(x["reason"])) == (DECLINED, R_OUT_SPACE)
                assert int(x["body_len"]) == len(host[i]["path"]) + len(host[i]["body"])
        if cap == 16:
            assert all(int(x["status"]) == DECLINED for x in res)


def test_mixed_call(ctx):
    rng = np.random.default_rng(6)
    mixed = [B.bedrock_chat(500 + i, int(rng.integers(1 << 10, 2 << 20)), bool(i % 2)) for i in range(8)] + [L.long_chat(60 + i, int(rng.integers(1 << 10, 1 << 20))) for i in range(4)]
    mixed += [G.W.diverse_body(s) for s in range(50)] + G.EDGES + G.ERRORS
    c = cfg(ctx, "ovr")
    whole = large(ctx, c, mixed)
    order = list(rng.permutation(len(mixed)))
    rev = large(ctx, c, [mixed[i] for i in order])
    cut = len(mixed) // 3
    split = large(ctx, c, mixed[:cut]) + large(ctx, c, mixed[cut:])
    for i, j in enumerate(order):
        assert all(rev[i][k] == whole[j][k] for k in KEYS)
    for a, b in zip(whole, split):
        assert all(a[k] == b[k] for k in KEYS)
    assert sum(g["status"] == OK for g in whole[:12]) == 12


def _mutations(seed, positions):
    out = []
    for p in positions:
        if p >= len(seed):
            continue
        out.append(seed[:p] + seed[p + 1:])
        out.append(seed[:p] + seed[p:p + 1] + seed[p:])
        for r in (b'"', b"\\", b"{", b"]", b",", b"0", b"x"):
            if seed[p:p + 1] != r:
                out.append(seed[:p] + r + seed[p + 1:])
    return out


def test_one_byte_mutations(ctx):
    """every deletion, duplication and replacement of each byte of the small seeds, and of each byte of a 20 KB seed near its
    thread, warp and tile edges: an OK is the oracle's record, every other status that is not a
    decline is the oracle's, and a decline has a reason"""
    small_seeds = [b for b in B.edge_requests()] + [b'{"model":"m","messages":[{"role":"tool","content":"a","tool_call_id":"i"},{"role":"tool","content":[{"type":"text","text":"b"}]}],"tools":[{"type":"function","function":{"name":"f","parameters":{"b":1,"a":[1,2]}}}]}']
    big = B.bedrock_chat(777, 2 << 10)
    # every byte within 40 of each warp (1 KiB) and tile (8 KiB) edge, and of each thread (32-byte) edge of the first warp
    edges = [e for e in range(1024, len(big), 1024)] + list(range(32, 1024, 32))
    positions = sorted({e + d for e in edges for d in range(-40, 41) if 0 <= e + d < len(big)})
    bodies = [m for s in small_seeds for m in _mutations(s, range(len(s)))] + _mutations(big, positions)
    c = cfg(ctx)
    got = [g for i in range(0, len(bodies), 4000) for g in large(ctx, c, bodies[i:i + 4000])]
    for b, g in zip(bodies, got):
        if g["status"] == DECLINED:
            assert g["reason"] != 0
            continue
        t = O.chat_translate("aws-bedrock", b)
        assert g["status"] == t.status, (b[:200], g["status"], g["reason"], t.status, t.err)
        if t.status == O.OK:
            assert g["path"].decode() == t.path and g["body"] == t.body, b[:200]
