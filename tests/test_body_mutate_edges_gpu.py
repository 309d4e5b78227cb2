"""body_mutate_kernel at its lane, round, member-pass, piece, copy-path, staging, class and capacity edges.  Every body is valid
JSON; its status and reason must be exactly what test_body_mutate_edges_cpu.expected_status says, an OK record must be the
oracle's bytes (oracle/mutate.hpp), and flags bit0 must say whether those bytes are the input's.  The generators live in
test_body_mutate_edges_cpu.py, which checks them without a GPU."""
import random

import numpy as np
import pytest

import _oracle as O
import test_body_mutate_edges_cpu as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gw():
    from aigw_b200 import capi
    g = capi.Context(0)
    yield g
    g.close()


def check_exact(gw, rm, st, bodies, max_len=None):
    """host form (16-aligned starts, max_len = the longest body): exact status, reason, bytes and flag for every body"""
    got = gw.body_mutate(rm, st, bodies)
    ml = max(len(b) for b in bodies) if max_len is None else max_len
    n_ok = 0
    for b, (status, reason, out, same) in zip(bodies, got):
        want = E.expected_status(b, rm, st, ml)
        assert (status, reason) == want, (b[:160], len(b), rm, st, status, reason, want)
        if status == E.OK:
            rc, exp = O.body_mutate(b, rm, st)
            assert rc == 0 and out == exp, (b[:160], rm, st, out[:200], exp[:200])
            assert same == (exp == b), (b[:160], rm, st)
            n_ok += 1
    return n_ok


def run_device(gw, rm, st, bodies, mods, max_len, out_cap=None, guard=512):
    """aigw_body_mutate_device over a hand-built arena: body i starts at an offset = mods[i] (mod 16).  Returns (results,
    record bytes per OK body, output guard bytes, out_used)."""
    from aigw_b200 import capi
    offs, pos = [], 0
    for b, m in zip(bodies, mods):
        pos = (pos + 15) // 16 * 16 + m
        offs.append(pos); pos += len(b) + 1
    arena = np.full(pos + 64, 0x7F, dtype=np.uint8)
    for b, o in zip(bodies, offs):
        arena[o:o + len(b)] = np.frombuffer(b, dtype=np.uint8)
    offs = np.asarray(offs, dtype=np.uint64); lens = np.asarray([len(b) for b in bodies], dtype=np.uint32)
    n = len(bodies)
    if out_cap is None:
        out_cap = sum((len(b) + 4096 + 15) // 16 * 16 for b in bodies)
    d_b = gw.dalloc(len(arena)); d_o = gw.dalloc(offs.nbytes); d_l = gw.dalloc(lens.nbytes)
    d_out = gw.dalloc(out_cap + guard); d_r = gw.dalloc(n * 16); d_u = gw.dalloc(64)
    try:
        gw.h2d(d_b, arena); gw.h2d(d_o, offs); gw.h2d(d_l, lens)
        gw.memset(d_out, 0xA5, out_cap + guard); gw.memset(d_r, 0xEE, n * 16)
        gw.body_mutate_device(rm, st, d_b, d_o, d_l, n, max_len, d_out, out_cap, d_r, d_u)
        gw.sync()
        res = np.zeros(n, dtype=capi.MutResult); gw.d2h(res, d_r)
        used = np.zeros(1, dtype=np.uint64); gw.d2h(used, d_u)
        out = np.zeros(out_cap + guard, dtype=np.uint8); gw.d2h(out, d_out)
    finally:
        for p in (d_b, d_o, d_l, d_out, d_r, d_u):
            gw.dfree(p)
    recs = [bytes(out[int(r["out_off"]):int(r["out_off"]) + int(r["out_len"])]) if r["status"] == 0 else None for r in res]
    return res, recs, out[out_cap:], int(used[0])


def check_device(gw, rm, st, bodies, mods, max_len):
    res, recs, guard, _ = run_device(gw, rm, st, bodies, mods, max_len)
    assert (guard == 0xA5).all()
    for b, r, rec in zip(bodies, res, recs):
        want = E.expected_status(b, rm, st, max_len)
        assert (int(r["status"]), int(r["reason"])) == want, (len(b), max_len, b[:100], int(r["status"]), int(r["reason"]), want)
        if want[0] == E.OK:
            exp = O.body_mutate(b, rm, st)[1]
            assert rec == exp and bool(int(r["flags"]) & 1) == (exp == b) and int(r["out_off"]) % 16 == 0


# ---------------------------------------------------------------- stage A and B at lane and round boundaries
@pytest.mark.parametrize("targets", [E.LANE_TARGETS + E.ROUND_TARGETS, E.BIG_TARGETS], ids=["5120-class", "17408-class"])
def test_adversarial_strings_at_lane_and_round_boundaries(gw, targets):
    bodies = [b for _k, _t, b, _o, _c in E.adversarial_corpus(targets)]
    for rm, st in E.ADV_MUTS:
        assert check_exact(gw, rm, st, bodies) == len(bodies)


def test_backslash_runs_in_values_and_keys(gw):
    vals = [b for *_x, b in E.runs_corpus(False)]
    keys = [b for *_x, b in E.runs_corpus(True)]
    for rm, st in [(["model"], []), ([], [("model", '"n"')]), (["a"], [("z", "1")])]:
        assert check_exact(gw, rm, st, vals) == len(vals)
        assert check_exact(gw, rm, st, keys) == 0          # every one AIGW_R_ESCAPE
    # both together in one call, so that warps see escaped keys and long runs in turn
    mixed = vals + keys
    random.Random(3).shuffle(mixed)
    check_exact(gw, ["model"], [], mixed)


def test_member_counts_positions_and_duplicates(gw):
    corpus = E.members_corpus()
    bodies = [b for *_x, b in corpus]
    for rm, st in E.MEMBER_MUTS:
        check_exact(gw, rm, st, bodies)
    r = gw.body_mutate(["e"], [], [E.members_body(128, (127,)), E.members_body(129, (127,)), E.members_body(64, (5, 40)), E.members_body(40, (3, 20))])
    assert [(x[0], x[1]) for x in r] == [(0, 0), (4, E.R_TOKENS), (4, E.R_DUP_KEY), (4, E.R_DUP_KEY)]


# ---------------------------------------------------------------- stage C: pieces, config text, copy paths, flags
def test_worst_case_pieces_are_ok(gw):
    body, cfgs = E.worst_pieces()
    for rm, st in cfgs:
        assert check_exact(gw, rm, st, [body, body[:-1] + b',"k00":"x"}']) == 1   # the second repeats k00: AIGW_R_DUP_KEY


def test_config_text_limit(gw):
    v = E.text_limit_value()
    bodies = [b'{"a":1,"b":2}', b'{"big":0,"a":[1]}', b'{"c":"' + b"c" * 300 + b'"}']
    assert check_exact(gw, ["a"], [("big", v)], bodies) == 3
    with pytest.raises(RuntimeError):
        gw.body_mutate(["a"], [("big", v[:-1] + 'v"')], bodies)


def test_copy_paths(gw):
    groups = {}
    for kind, d, L, body, rm, st in E.copy_corpus():
        groups.setdefault((tuple(rm), tuple(st)), []).append(body)
    for (rm, st), bodies in groups.items():
        assert check_exact(gw, list(rm), list(st), bodies) == len(bodies)


def test_unchanged_flag(gw):
    for body, rm, st in E.FLAG_CASES:
        (status, reason, out, same), = gw.body_mutate(rm, st, [body])
        exp = O.body_mutate(body, rm, st)[1]
        assert status == 0 and out == exp and same == (exp == body), (body, rm, st, same)
    assert gw.body_mutate([], [("a", "1")], [b'{"a":1}'])[0][3]
    assert gw.body_mutate(["a"], [("a", "1")], [b'{"b":2,"a":1}'])[0][3]
    assert not gw.body_mutate([], [("a", "2")], [b'{"a":1}'])[0][3]


# ---------------------------------------------------------------- staging, size classes, capacity
def test_staging_offsets_and_classes(gw):
    small = [b for _k, _t, b, _o, _c in E.adversarial_corpus(E.LANE_TARGETS)][:16] + [E.exact_len_body(n) for n in (100, 1025, 4097)]
    big = [E.exact_len_body(n) for n in E.CLASS_LENS] + [E.exact_len_body(n) for n in (9000, 30000)]
    rm, st = ["model"], [("t", "2"), ("new", '"v"')]
    for max_len in (5120, 9000, 17408, 65536, 70000):
        bodies = small + big
        for shift in (0, 5):
            mods = [(i + shift) % 16 for i in range(len(bodies))]
            check_device(gw, rm, st, bodies, mods, max_len)
    # every class from the host form too: a call's longest body picks it
    for top in (5120, 9000, 17408, 65536):
        bodies = [b for b in small + big if len(b) <= top]
        assert max(len(b) for b in bodies) == top
        assert check_exact(gw, rm, st, bodies) == len(bodies)


@pytest.mark.parametrize("cls", [5120, 17408, 65536])
def test_output_capacity(gw, cls):
    rm, st = ["model"], [("t", "22")]
    sizes = [s for s in (60, 700, 3000, 5000, 12000, 40000) if s <= cls]
    bodies = [E.exact_len_body(s) for s in sizes] * 12
    mods = [i % 16 for i in range(len(bodies))]
    exps = [O.body_mutate(b, rm, st)[1] for b in bodies]
    exact = sum((len(e) + 15) // 16 * 16 for e in exps)
    for cap in (exact, exact - 1):
        res, recs, guard, used = run_device(gw, rm, st, bodies, mods, cls, out_cap=cap)
        assert (guard == 0xA5).all() and used == exact
        st_ = [int(r["status"]) for r in res]
        for r, rec, exp in zip(res, recs, exps):
            if int(r["status"]) == 0:
                assert rec == exp and int(r["out_off"]) + int(r["out_len"]) <= cap
            else:
                assert int(r["reason"]) == E.R_ARENA_FULL
        if cap == exact:
            assert st_ == [0] * len(bodies)
        else:
            assert st_.count(4) >= 1 and st_.count(0) >= 1


# ---------------------------------------------------------------- mixed batches through the persistent loop
def _mixed(rng, limit):
    pool = [b for _k, _t, b, _o, _c in E.adversarial_corpus(E.LANE_TARGETS + E.ROUND_TARGETS + E.BIG_TARGETS)]
    pool += [b for *_x, b in E.runs_corpus(False)] + [b for *_x, b in E.runs_corpus(True)]
    pool += [b for *_x, b in E.members_corpus()]
    pool += [E.exact_len_body(n) for n in E.CLASS_LENS]
    pool += [b'{"model":"m", "x":1}', b'{"model":"m","model":"n"}', b'{"\\u006dodel":1}', b'{}', b'{ }', b'{"x":{"model" : 1}}']
    pool = [b for b in pool if len(b) <= limit]
    return [rng.choice(pool) for _ in range(4000)]


@pytest.mark.parametrize("limit", [5120, 17408, 70000])
def test_mixed_batch(gw, limit):
    rng = random.Random(limit)
    bodies = _mixed(rng, limit)
    for rm, st in [(["model"], []), (["x"], [("model", '"gpt"'), ("extra", "[1,2]")])]:
        got = gw.body_mutate(rm, st, bodies)
        ml = max(len(b) for b in bodies)
        cache = {}
        kinds = set()
        for b, (status, reason, out, same) in zip(bodies, got):
            want = E.expected_status(b, rm, st, ml)
            assert (status, reason) == want, (b[:120], status, reason, want)
            kinds.add(reason)
            if status == 0:
                if b not in cache:
                    cache[b] = O.body_mutate(b, rm, st)[1]
                assert out == cache[b] and same == (cache[b] == b)
        assert {E.R_NONE, E.R_ESCAPE} <= kinds and len(kinds) >= 3
