"""BASELINE config 3 at its edges: bpe_count_kernel at its staging, group and table edges, emb_scan_kernel at its thread, warp and
tile boundaries and at both capacities of a call.  Every count is exact: a text is declined exactly when the decline rule of
test_config3_edges_cpu.py says so, and otherwise its count is the BPE oracle's (oracle/bpe.hpp); a request's verdict is the
embeddings oracle's (oracle/embeddings.hpp) or a decline this file names.  The generators live in test_config3_edges_cpu.py,
which checks them without a GPU."""
import json
import os

import numpy as np
import pytest

import _oracle as O
import test_config3_edges_cpu as E

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
VOCAB = json.load(open(os.path.join(HERE, "golden", "bpe_vocab.json")))
OK, MALFORMED_400, DECLINED = 0, 1, 4


@pytest.fixture(scope="module")
def gw():
    from aigw_b200 import capi
    g = capi.Context(0)
    g.bpe = g.bpe_load(VOCAB["byte_to_id"], VOCAB["merges"])
    g.orc = O.Bpe(VOCAB)
    yield g
    g.bpe_free(g.bpe)
    g.close()


# ---------------------------------------------------------------- BPE count
def pack_texts(texts, base=0):
    lens = np.asarray([len(t) for t in texts], dtype=np.uint32)
    offs = np.zeros(len(texts), dtype=np.uint64)
    if len(texts) > 1:
        offs[1:] = np.cumsum(lens[:-1], dtype=np.uint64)
    offs += base
    arena = np.frombuffer(b"\x7f" * base + b"".join(texts) + b"\0" * 16, dtype=np.uint8).copy()
    return arena, offs, lens


def bpe_device(g, bpe, texts):
    arena, offs, lens = pack_texts(texts)
    n = len(texts)
    ptrs = [g.dalloc(arena.nbytes), g.dalloc(offs.nbytes), g.dalloc(lens.nbytes), g.dalloc(4 * n)]
    try:
        g.h2d(ptrs[0], arena); g.h2d(ptrs[1], offs); g.h2d(ptrs[2], lens)
        g.bpe_count_device(bpe, ptrs[0], ptrs[1], ptrs[2], n, ptrs[3])
        out = np.zeros(n, dtype=np.uint32); g.d2h(out, ptrs[3])
    finally:
        for p in ptrs:
            g.dfree(p)
    return out


def check_counts(g, bpe, orc, texts, device=False):
    """Host form (and the device form when asked) against the decline rule and the oracle: no declines beyond the rule."""
    got = g.bpe_count(bpe, texts)
    if device:
        assert np.array_equal(bpe_device(g, bpe, texts), got)
    exp = orc.count(texts)
    for i, (t, x, e) in enumerate(zip(texts, got, exp)):
        if E.declined(t):
            assert int(x) == E.DECLINED, (i, len(t), [len(p) for p in E.pieces(t)][:8])
        else:
            assert int(x) == int(e), (i, len(t), t[:60], int(x), int(e))
    return got


def test_staging_texts(gw):
    t = E.staging_texts()
    got = check_counts(gw, gw.bpe, gw.orc, t, device=True)
    assert (got == E.DECLINED).sum() > 20 and (got != E.DECLINED).sum() > 500
    check_counts(gw, gw.bpe, gw.orc, t[::-1])


def test_piece_of_512_bytes_is_counted_anywhere(gw):
    t = E.decline_texts()
    got = check_counts(gw, gw.bpe, gw.orc, t, device=True)
    assert any(int(x) != E.DECLINED and any(len(p) == E.BUF for p in E.pieces(s)[:-1]) for s, x in zip(t, got))
    for s in t:                       # one text per call: the text starts its own group
        check_counts(gw, gw.bpe, gw.orc, [s])


def test_buffer_fill(gw):
    for total, k, texts in E.fill_calls():
        check_counts(gw, gw.bpe, gw.orc, texts)


def test_group_sizes_and_long_texts(gw):
    for texts in E.group_calls():
        check_counts(gw, gw.bpe, gw.orc, texts)


def vocab_texts(vocab, seed, n=600):
    """Texts over the bytes the vocabulary merges, with spaces, lengths 0 .. 1100 (some pieces longer than the buffer)."""
    r = np.random.default_rng(seed)
    alpha = sorted({m[k] for m in vocab["merges"] for k in (0, 1) if m[k] < 256} | {c for c in range(256) if vocab["byte_to_id"][c] != c})
    alpha = [c for c in alpha if c != 0x20] or [ord("a")]
    out = []
    for i in range(n):
        L = int(r.choice([0, 1, 2, 3, 7, 40, 200, 511, 512, 513, 700, 1100]))
        space = float(r.choice([0.0, 0.02, 0.2]))
        b = bytes(0x20 if r.random() < space else alpha[int(r.integers(len(alpha)))] for _ in range(L))
        out.append(b)
    return out


SYNTHETIC = {
    "binary_chain_9": lambda: E.chain_vocab_binary(9),
    "linear_chain_512": lambda: E.chain_vocab_linear(512),
    "linear_chain_7": lambda: E.chain_vocab_linear(7),
    "collisions": lambda: E.collision_vocab()[0],
    "largest_4096": lambda: E.largest_vocab(4096),
    "high_ids": E.high_id_vocab,
    "duplicates": E.duplicate_vocab,
}


@pytest.mark.parametrize("name", list(SYNTHETIC))
def test_synthetic_vocabulary(gw, name):
    vocab = SYNTHETIC[name]()
    bpe = gw.bpe_load(vocab["byte_to_id"], vocab["merges"])
    try:
        orc = O.Bpe(vocab)
        texts = vocab_texts(vocab, seed=len(name))
        texts += [b"a" * n for n in range(0, 1100, 7)] + [b"a" * n + b" " + b"a" * m for n, m in ((511, 511), (512, 511), (100, 512), (1, 513))]
        if name == "collisions":
            pairs = E.collision_vocab()[1]
            texts += [bytes(p) for p in pairs] + [b"".join(bytes(p) for p in pairs)] + [b" ".join(bytes(p) for p in pairs)]
        got = check_counts(gw, bpe, orc, texts, device=True)
        if name == "collisions":   # every colliding pair, the one probed into slot `mask` and the wrapped ones too, merges
            assert all(int(x) == 1 for x in got[-11:-2])
    finally:
        gw.bpe_free(bpe)


def test_load_limits(gw):
    big = E.largest_vocab(4096)
    bpe = gw.bpe_load(big["byte_to_id"], big["merges"]); gw.bpe_free(bpe)
    over = E.largest_vocab(4097)
    with pytest.raises(RuntimeError):
        gw.bpe_load(over["byte_to_id"], over["merges"])
    top = E.high_id_vocab()
    bpe = gw.bpe_load(top["byte_to_id"], top["merges"]); gw.bpe_free(bpe)
    for where in ("byte", "a", "b", "merged"):
        b2i = list(top["byte_to_id"]); merges = [list(m) for m in top["merges"]]
        if where == "byte":
            b2i[ord("q")] = 65535
        else:
            merges[1][("a", "b", "merged").index(where)] = 65535
        with pytest.raises(RuntimeError):
            gw.bpe_load(b2i, merges)


# ---------------------------------------------------------------- embeddings requests
def emb_device(g, bpe, bodies, max_len=None, total_bytes=None):
    from aigw_b200 import capi
    arena, offs, lens = capi.pack_bodies(bodies)
    n = len(bodies)
    ptrs = [g.dalloc(arena.nbytes), g.dalloc(offs.nbytes), g.dalloc(lens.nbytes), g.dalloc(32 * n)]
    try:
        g.h2d(ptrs[0], arena); g.h2d(ptrs[1], offs); g.h2d(ptrs[2], lens)
        g.embeddings_count_device(bpe, ptrs[0], ptrs[1], ptrs[2], n, int(lens.max()) if max_len is None else max_len,
                                  arena.nbytes if total_bytes is None else total_bytes, ptrs[3])
        res = np.zeros(n, dtype=capi.EmbCountResult); g.d2h(res, ptrs[3])
    finally:
        for p in ptrs:
            g.dfree(p)
    return res


def check_requests(g, bodies, res, declines=None):
    """Every result against the oracle; `declines` maps a body index to the reason of the decline it must get."""
    declines = declines or {}
    n_ok = 0
    for i, (b, x) in enumerate(zip(bodies, res)):
        if i in declines:
            assert (int(x["status"]), int(x["reason"])) == (DECLINED, declines[i]), (i, len(b), x)
            continue
        t = O.embeddings_translate("openai", b)
        assert int(x["status"]) == t.status, (i, len(b), b[:80], x, t.err)
        if t.status != OK:
            continue
        texts = E.request_inputs(b)
        assert int(x["n_inputs"]) == len(texts), (i, x)
        mo, ml = int(x["model_off"]), int(x["model_len"])
        assert b[mo:mo + ml] == t.model, (i, b[mo:mo + ml], t.model)
        dec = [E.declined(s) for s in texts]
        kept = [s for s, d in zip(texts, dec) if not d]
        assert int(x["declined_inputs"]) == sum(dec), (i, x)
        assert int(x["tokens"]) == int(np.asarray(g.orc.count(kept), dtype=np.uint64).sum()) if kept else int(x["tokens"]) == 0, (i, x)
        n_ok += 1
    return n_ok


@pytest.mark.parametrize("feature", E.FEATURES)
def test_feature_at_boundaries(gw, feature):
    bodies = [b for b in (E.feature_body(feature, p) for p in E.feature_positions()) if b is not None]
    res = gw.embeddings_count(gw.bpe, bodies)
    reason = E.DECLINE_FEATURES.get(feature)
    n_ok = check_requests(gw, bodies, res, {i: reason for i in range(len(bodies))} if reason else None)
    if reason is None and feature not in ("true", "ctrl_outside"):
        assert n_ok == len(bodies)
    if feature in ("true", "ctrl_outside"):
        assert (res["status"] == MALFORMED_400).all()


def length_bodies():
    ls = [E.TILE * k + d for k in (1, 2, 3, 4) for d in (-1, 0, 1)]
    ls += [200 + r for r in range(32)] + [E.TILE - 32 + r for r in range(32)] + [2 * E.TILE + 64 + r for r in range(32)]
    bodies = [E.body_of_length(n, n) for n in ls]
    # trailing whitespace across a tile boundary, and inputs longer than one tile and than several
    bodies += [E.body_of_length(8100) + b" " * 200, E.body_of_length(8150) + b" \n\t\r" * 30 + b"\n", E.body_of_length(16383) + b" "]
    bodies += [b'{"input":"' + E.pad(20000) + b'"}', b'{"model":"m","input":["' + E.pad(50000, 3) + b'","' + E.pad(9000, 5) + b'"]}']
    return bodies


def test_body_lengths_host_and_device(gw):
    bodies = length_bodies()
    res = gw.embeddings_count(gw.bpe, bodies)
    assert check_requests(gw, bodies, res) == len(bodies)
    dev = emb_device(gw, gw.bpe, bodies)
    for f in res.dtype.names:
        if f != "first_text":       # the row of a request's first input depends on the order CTAs take requests in
            assert np.array_equal(dev[f], res[f]), f


def test_sixteen_mib(gw):
    """16 MiB - 1 bytes are accepted, 16 MiB are TOO_LARGE.  The device form with a small max_len keeps the token workspace small
    (the request has 7 scan tokens)."""
    n = (1 << 24) - 1
    ok = b'{"input":["' + E.pad(n - 14) + b'"]}'
    big = b'{"input":["' + E.pad(n - 13) + b'"]}'
    assert len(ok) == n and len(big) == n + 1
    res = emb_device(gw, gw.bpe, [ok, big], max_len=4096)
    assert int(res[0]["status"]) == OK and int(res[0]["n_inputs"]) == 1 and int(res[0]["declined_inputs"]) == 0
    assert int(res[0]["tokens"]) == int(gw.orc.count([E.pad(n - 14)])[0])
    assert (int(res[1]["status"]), int(res[1]["reason"])) == (DECLINED, E.R_TOO_LARGE)


def test_token_capacity(gw):
    """tok_cap = max_len / 2 + 64 scan tokens per request: exactly tok_cap is counted, one more is AIGW_R_TOKENS."""
    for L in (484, 1000, 6001, 20000):
        cap = L // 2 + 64
        at, over = E.tokens_body(cap, L), E.tokens_body(cap + 1, L)
        assert E.scan_tokens(at) == cap and E.scan_tokens(over) == cap + 1
        res = gw.embeddings_count(gw.bpe, [at])
        check_requests(gw, [at], res)
        assert int(res[0]["status"]) == OK
        res = gw.embeddings_count(gw.bpe, [over])
        check_requests(gw, [over], res, {0: E.R_TOKENS})
    # max_len set by a larger neighbour in the same call
    M = 9000
    cap = M // 2 + 64
    filler = E.body_of_length(M)
    at, over = E.tokens_body(cap, cap + 300), E.tokens_body(cap + 1, cap + 300)
    res = gw.embeddings_count(gw.bpe, [at, filler, over])
    check_requests(gw, [at, filler, over], res, {2: E.R_TOKENS})
    assert int(res[0]["status"]) == OK


def dense_body(m, seed):
    """m inputs, mostly empty strings (3 bytes and 3 tokens each); every 50th holds a few words."""
    items = [b'"' + E.words_text(9, seed + i) + b'"' if i % 50 == 0 else b'""' for i in range(m)]
    return b'{"input":[' + b",".join(items) + b"]}"


def test_text_table_capacity(gw):
    """The call's text table has total_bytes / 4 + 1024 rows.  Dense requests (one row per 3 bytes), admitted by the token capacity
    a large neighbour sets, overflow it: each request is exact or AIGW_R_ARENA_FULL, the accepted rows fit, and a following call
    is unaffected.  Which request fails depends on the order in which CTAs reach them."""
    big = b'{"input":"' + E.pad(65536 - 13) + b'"}'
    bodies = [big] + [dense_body(10000, 100 * k) for k in range(12)]
    from aigw_b200 import capi
    arena, offs, lens = capi.pack_bodies(bodies)
    cap = arena.nbytes // 4 + 1024
    assert sum(len(E.request_inputs(b)) for b in bodies) > cap
    for _ in range(2):
        res = emb_device(gw, gw.bpe, bodies)
        full = {i for i, x in enumerate(res) if int(x["status"]) == DECLINED}
        assert full and len(full) < len(bodies) - 1
        check_requests(gw, bodies, res, {i: E.R_ARENA_FULL for i in full})
        assert int(res["n_inputs"][res["status"] == OK].astype(np.int64).sum()) <= cap
    after = length_bodies()[:20]
    assert check_requests(gw, after, gw.embeddings_count(gw.bpe, after)) == 20


def test_declined_inputs_are_exact(gw):
    inputs = [E.words_text(n, n) for n in (0, 5, 511, 512, 513, 1500)] + [b"x" * n for n in (511, 512, 513, 2000)]
    inputs += [b"y " + b"x" * n for n in (510, 511, 512)] + [E.words_text(600, 1) + b" " + b"z" * n + b" w" for n in (510, 511, 512)]
    bodies = [b'{"model":"m","input":[' + b",".join(b'"' + s + b'"' for s in inputs[k:] + inputs[:k]) + b"]}" for k in range(len(inputs))]
    bodies += [b'{"input":"' + s + b'"}' for s in inputs]
    res = gw.embeddings_count(gw.bpe, bodies)
    assert check_requests(gw, bodies, res) == len(bodies)
    assert (res["declined_inputs"][:len(inputs)] == sum(E.declined(s) for s in inputs)).all()


def test_many_requests_no_state_carries_over(gw):
    """Far more requests than CTAs, errors, declines and capacity declines interleaved with OK requests, so that every CTA
    handles an OK request right after a failed one."""
    kinds = []
    bodies = []
    for i in range(3000):
        k = i % 6
        p = 40 + (i * 97) % 9000
        if k == 0:
            bodies.append(E.feature_body("backslash", p)); kinds.append(E.R_ESCAPE)
        elif k == 1:
            bodies.append(E.feature_body("true", p)); kinds.append(None)
        elif k == 2:
            bodies.append(E.feature_body("ctrl_in_string", p)); kinds.append(E.R_CTRL_IN_STRING)
        elif k == 3:
            bodies.append(b'{"input":["' + b'"' * 3); kinds.append(None)          # unterminated: 400
        else:
            bodies.append(E.feature_body("close_quote" if k == 4 else "dimensions", p)); kinds.append(None)
    res = gw.embeddings_count(gw.bpe, bodies)
    declines = {i: r for i, r in enumerate(kinds) if r is not None}
    assert check_requests(gw, bodies, res, declines) == 1000


def test_host_offsets_out_of_order_and_arena_base(gw):
    from aigw_b200 import capi
    bodies = length_bodies()[:40] + [E.feature_body("utf8", 8192 + d) for d in range(-5, 5)]
    want = gw.embeddings_count(gw.bpe, bodies)
    # the same bodies in reverse order inside an arena that starts 4096 bytes after its base
    arena0, offs0, lens = capi.pack_bodies(bodies)
    order = np.arange(len(bodies))[::-1]
    pos = np.zeros(len(bodies), dtype=np.uint64)
    cur = 4096
    for i in order:
        pos[i] = cur
        cur += (int(lens[i]) + 15) // 16 * 16
    arena = np.full(cur + 16, 0x20, dtype=np.uint8)
    for i, b in enumerate(bodies):
        arena[int(pos[i]):int(pos[i]) + len(b)] = np.frombuffer(b, dtype=np.uint8)
    res, _ = gw.embeddings_count_host(gw.bpe, arena, pos, lens)
    for f in ("status", "reason", "n_inputs", "tokens", "declined_inputs", "model_len", "in_len"):
        assert np.array_equal(res[f], want[f]), f
    assert np.array_equal(res["model_off"], want["model_off"])
