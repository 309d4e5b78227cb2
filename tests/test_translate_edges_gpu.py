"""The chat translate pass at its layout edges: exact size-class lengths, the token capacity kTok, features that straddle lane and
round boundaries, nesting depth, and a structural mutation corpus.  Every case runs through the throughput pipeline, the fused
small-batch kernel (bodies ≤ 5120 bytes) and the device-resident call (exact max_len and max_len = 0); every path must agree
with the others and with the oracle.  The generators live in test_translate_edges_cpu.py, which checks them without a GPU.

Contract (as in test_chat_gpu.py): GPU OK ⇒ oracle OK with identical body, path, model span, stream flag and body kind; an error
status is the oracle's status; DECLINED only where a test allows it.  A capacity decline (tokens, ops, scratch) may differ
between paths whose size classes differ: the path with the smaller class may leave a body to the stock path that a larger
class translates, and the oracle decides the larger class's answer."""
import collections
import time

import numpy as np
import pytest

import _oracle as O
import test_translate_edges_cpu as E

pytestmark = pytest.mark.gpu

OK, DECLINED = 0, 4


@pytest.fixture(scope="module")
def ctx():
    import aigw_b200 as A
    c = A.Context(0)
    yield c
    c.chat_set_small_batch(-1)
    c.close()


def cfg_of(ctx, schema):
    return ctx.cfg(schema, prefix="v1" if schema == "msg-openai" else None)


def device_translate(ctx, cfg, bodies, max_len):
    """aigw_chat_translate_device on device copies of `bodies`; results in the format of Context.chat_translate"""
    import aigw_b200 as A
    n = len(bodies)
    arena, offs, lens = A.capi.pack_bodies(bodies)
    out_cap = 2 * int(lens.astype(np.int64).sum()) + 1024 * n + 4096
    ptrs = []
    try:
        d_in, d_off, d_len = ctx.dalloc(arena.nbytes), ctx.dalloc(offs.nbytes), ctx.dalloc(lens.nbytes)
        ptrs += [d_in, d_off, d_len]
        d_out, d_res, d_used = ctx.dalloc(out_cap), ctx.dalloc(n * 32), ctx.dalloc(8)
        ptrs += [d_out, d_res, d_used]
        ctx.h2d(d_in, arena); ctx.h2d(d_off, offs); ctx.h2d(d_len, lens); ctx.memset(d_used, 0, 8)
        ctx.chat_translate_device(cfg, d_in, d_off, d_len, n, max_len, d_out, out_cap, d_res, d_used)
        res = np.zeros(n, dtype=A.DocResult); ctx.d2h(res, d_res)
        used = np.zeros(1, dtype=np.uint64); ctx.d2h(used, d_used)
        out = np.zeros(max(16, int(used[0])), dtype=np.uint8); ctx.d2h(out, d_out, int(used[0]))
    finally:
        for p in ptrs:
            ctx.dfree(p)
    return [to_dict(res[i], out, bodies[i]) for i in range(n)]


def to_dict(x, out, body):
    o = int(x["out_off"]); pl = int(x["path_len"]); bl = int(x["body_len"]); ok = int(x["status"]) == OK
    return {"status": int(x["status"]), "reason": int(x["reason"]), "path": bytes(out[o:o + pl]) if ok else b"", "body": bytes(out[o + pl:o + pl + bl]) if ok else b"",
            "model": body[int(x["model_off"]):int(x["model_off"]) + int(x["model_len"])], "stream": bool(x["flags"] & 1), "body_kind": int(x["body_kind"])}


def run_paths(ctx, schema, bodies):
    """{path name: (class of each body in that path, results)}"""
    return run_cfg_paths(ctx, cfg_of(ctx, schema), bodies)


def run_cfg_paths(ctx, cfg, bodies):
    """run_paths under a backend configuration of the caller's"""
    paths = {}
    try:
        ctx.chat_set_small_batch(0)
        paths["pipeline"] = ([E.class_of(len(b)) for b in bodies], ctx.chat_translate(cfg, bodies))
        small = [i for i, b in enumerate(bodies) if 0 < len(b) <= E.SMALL_MAX]
        if small:
            ctx.chat_set_small_batch(1 << 20)
            got = ctx.chat_translate(cfg, [bodies[i] for i in small])
            r = [None] * len(bodies)
            for i, g in zip(small, got):
                r[i] = g
            paths["fused"] = ([E.SMALL_MAX] * len(bodies), r)
    finally:
        ctx.chat_set_small_batch(-1)
    groups = collections.defaultdict(list)
    for i, b in enumerate(bodies):
        groups[E.class_of(len(b))].append(i)
    r = [None] * len(bodies); cls = [0] * len(bodies)
    for c, idx in groups.items():   # one call per class, max_len = the longest body of the call
        got = device_translate(ctx, cfg, [bodies[i] for i in idx], max(len(bodies[i]) for i in idx))
        for i, g in zip(idx, got):
            r[i] = g; cls[i] = c
    paths["device"] = (cls, r)
    paths["device_max0"] = ([E.CLASSES[-1]] * len(bodies), device_translate(ctx, cfg, bodies, 0))
    return paths


def check_contract(schema, body, g, o, where):
    if g["status"] == OK:
        assert o.status == O.OK, (where, body[:300], o.err)
        exp = o.body if o.body_kind == O.BYTES else b""
        assert g["body"] == exp, (where, body[:300], g["body"][:300], exp[:300])
        assert g["path"].decode() == o.path and g["model"] == o.model and g["stream"] == o.stream and g["body_kind"] == o.body_kind, (where, body[:300], g, o.path)
    elif g["status"] != DECLINED:
        assert g["status"] == o.status, (where, body[:300], g, o.status, o.err)


def check_paths(schema, bodies, paths):
    """every path against the oracle, and the paths against each other; returns the oracle's results"""
    names = list(paths)
    oracle = []
    for i, b in enumerate(bodies):
        o = E.oracle(schema, b)
        oracle.append(o)
        for nm in names:
            g = paths[nm][1][i]
            if g is not None:
                check_contract(schema, b, g, o, (nm, i))
        for a in names:
            for c in names:
                ca, ga = paths[a][0][i], paths[a][1][i]
                cc, gc = paths[c][0][i], paths[c][1][i]
                if a >= c or ga is None or gc is None or ga == gc:
                    continue
                lo, hi = (ga, gc) if ca < cc else (gc, ga) if cc < ca else (None, None)
                assert lo is not None and lo["status"] == DECLINED and lo["reason"] in E.CAPACITY_REASONS, (i, a, c, b[:300], ga, gc)
    return oracle


def statuses(paths, i):
    return {nm: (r[i]["status"], r[i]["reason"]) for nm, (_, r) in paths.items() if r[i] is not None}


# ---------------------------------------------------------------- A1: exact size-class lengths
@pytest.mark.parametrize("schema", ["aws-bedrock", "openai", "gcp-vertexai", "msg-openai"])
def test_exact_size_class_lengths(ctx, schema):
    bodies = E.size_class_bodies(schema) + [E.too_large_body(schema)]
    if schema == "aws-bedrock":
        bodies += E.aligned_output_bodies()
    paths = run_paths(ctx, schema, bodies)
    check_paths(schema, bodies, paths)
    for i, b in enumerate(bodies):
        for nm, (st, reason) in statuses(paths, i).items():
            if len(b) > E.CLASSES[-1]:
                assert (st, reason) == (DECLINED, E.REASON_TOO_LARGE), (nm, len(b))
            else:
                assert st == OK, (nm, len(b), st, reason)


# ---------------------------------------------------------------- A2: token capacity
def test_token_capacity(ctx):
    cases = E.token_cases()
    bodies = [b for _, _, b in cases]
    paths = run_paths(ctx, "openai", bodies)
    oracle = check_paths("openai", bodies, paths)
    assert all(o.status == O.OK for o in oracle)
    pipe, fused = paths["pipeline"][1], paths["fused"][1]
    for (c, t, b), g, f, o in zip(cases, pipe, fused, oracle):
        cap = E.KTOK[E.class_of(len(b))]
        if t <= cap:
            assert g["status"] == OK, (c, t, g)
        else:
            assert (g["status"], g["reason"]) == (DECLINED, E.REASON_TOKENS), (c, t, g)
        if f is not None:
            if t <= E.SMALL_KTOK:
                assert f["status"] == OK, (c, t, f)
            else:
                assert (f["status"], f["reason"]) == (DECLINED, E.REASON_TOKENS), (c, t, f)
    # the 2048-class bodies with 640 tokens: the pipeline leaves them to the stock path, the fused kernel translates them
    assert any(c == 2048 and t == 640 and g["status"] == DECLINED and f["status"] == OK for (c, t, _), g, f in zip(cases, pipe, fused))


# ---------------------------------------------------------------- A3: straddles across lane, round and chunk boundaries
@pytest.mark.parametrize("schema", ["aws-bedrock", "openai"])
def test_boundary_straddles(ctx, schema):
    cases = E.straddle_cases()
    bodies = [b for _, _, _, b in cases]
    t0 = time.time()
    paths = run_paths(ctx, schema, bodies)
    check_paths(schema, bodies, paths)
    declined = collections.Counter()
    for i, (c, bnd, f, b) in enumerate(cases):
        for nm, (st, reason) in statuses(paths, i).items():
            if st != OK:
                declined[(nm, c, bnd, f, st, reason)] += 1
    print(schema, len(bodies), "bodies in %.1f s" % (time.time() - t0), "not OK:", dict(declined))
    assert not declined


@pytest.mark.parametrize("schema", ["aws-bedrock", "openai"])
def test_long_strings_respelled_escape_mask(ctx, schema):
    """a re-spelled escape only in the first or only in the last 32-byte block of a string that spans several mask words"""
    cases = E.long_string_cases()
    bodies = [b for _, _, b in cases]
    paths = run_paths(ctx, schema, bodies)
    check_paths(schema, bodies, paths)
    for i, (where, shift, b) in enumerate(cases):
        for nm, (st, reason) in statuses(paths, i).items():
            assert st == OK, (nm, where, shift, st, reason)


# ---------------------------------------------------------------- A4: nesting depth
# the deepest accepted nesting of each member: the index grammar check allows 48 open brackets in the document, the re-emit of a
# JSON value (tool arguments, Gemini parameters) 24 open containers below the value's root
MAX_DEPTH = {"passthrough": 47, "tool_args": 23, "gemini_params": 21}


@pytest.mark.parametrize("kind", list(E.DEPTH_SCHEMA))
def test_nesting_depth(ctx, kind):
    schema = E.DEPTH_SCHEMA[kind]
    ks = list(range(1, 61))
    bodies = [E.depth_body(kind, k) for k in ks]
    paths = run_paths(ctx, schema, bodies)
    oracle = check_paths(schema, bodies, paths)
    assert all(o.status == O.OK for o in oracle)
    for nm, (_, res) in paths.items():
        ok = [k for k, g in zip(ks, res) if g["status"] == OK]
        assert ok == list(range(1, ok[-1] + 1)), (nm, ok)
        assert ok[-1] == MAX_DEPTH[kind], (nm, kind, ok[-1])
        g = res[ks.index(MAX_DEPTH[kind] + 1)]
        assert (g["status"], g["reason"]) == (DECLINED, E.REASON_DEPTH), (nm, g)
        assert all(g["status"] == DECLINED for g in res[MAX_DEPTH[kind]:]), nm


# ---------------------------------------------------------------- regression: \u without four hex digits
INVALID_U_ESCAPES = [   # found by the mutation corpus: a key the walk skips was never decoded, so its bad escape went unnoticed
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"tempera\\ure":0.5,"top_p":1,"stop":["a","b"],"stream":true}',
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"x_key":"\\u12"}',
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"x_key":"\\u12g4"}',
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"x\\uZZZZ":1}',
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"x_key":{"\\u00":[1]}}',
    b'{"model":"m","messages":[{"role":"user","content":"x\\u00e"}]}',
    b'{"model":"m","messages":[{"role":"user","content":"x"}],"x_key":"\\u',
]


@pytest.mark.parametrize("schema", ["aws-bedrock", "openai", "gcp-vertexai"])
def test_invalid_unicode_escape_is_never_ok(ctx, schema):
    valid = b'{"model":"m","messages":[{"role":"user","content":"x"}],"x_key":"\\u00e9\\uABcd"}'
    bodies = INVALID_U_ESCAPES + [valid]
    paths = run_paths(ctx, schema, bodies)
    oracle = check_paths(schema, bodies, paths)
    for i, o in enumerate(oracle[:-1]):
        assert o.status == O.MALFORMED_400, (i, o.status)
        for nm, (st, reason) in statuses(paths, i).items():
            assert st != OK, (nm, bodies[i])
    assert oracle[-1].status == O.OK and all(st == OK for st, _ in statuses(paths, len(bodies) - 1).values())


# ---------------------------------------------------------------- A5: structural mutation corpus
def test_structural_mutations(ctx):
    by_schema = collections.defaultdict(list)
    for schema, b in E.mutation_seeds():
        by_schema[schema] += list(E.mutants(b))
    total = collections.Counter()
    for schema, bodies in by_schema.items():
        paths = run_paths(ctx, schema, bodies)
        oracle = check_paths(schema, bodies, paths)
        for g, o in zip(paths["pipeline"][1], oracle):
            total["mutants"] += 1
            total["oracle_400"] += o.status == O.MALFORMED_400
            total["oracle_ok"] += o.status == O.OK
            total["gpu_ok"] += g["status"] == OK
            total["gpu_400"] += g["status"] == 1
            total["gpu_declined"] += g["status"] == DECLINED
            total["gpu_other_error"] += g["status"] not in (OK, 1, DECLINED)
    print("mutation corpus:", dict(total))
    assert total["mutants"] > 20000
    assert total["oracle_400"] > total["mutants"] // 2   # the corpus reaches the grammar errors
