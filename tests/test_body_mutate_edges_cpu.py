"""Generators for the body-mutation edge tests (test_body_mutate_edges_gpu.py) and their self-checks (no GPU).

body_mutate_kernel<MAXD, W> (aigw_b200/csrc/mutate_kernel.cu) works in fixed units:
  stage A   one warp per body; per 1 KiB round each lane classifies 32 bytes.  The escape carry (odd backslash runs) and the
            string-parity carry cross lanes and rounds; a warp prefix sum gives each lane its brace depth
  stage B   one lane per top-level member, 32 members per pass, at most 128 members
  stage C   lane 0 folds the member actions into at most 96 copy pieces: maximal input runs, replacement values and appended
            members from the shared-memory config text, and the ',' the host puts at text[3068]
  copy      a piece of 64 bytes or more whose source and destination agree modulo 4 is copied by words after a head of
            (4 - dst & 3) & 3 bytes; every other piece byte by byte
  staging   16-byte loads when the body's start is 16-aligned, byte loads otherwise
  classes   (5120, 4 warps), (17408, 2), (65536, 1), picked by the call's max_len
The helpers here restate the decline list, the config text layout and the piece fold in plain Python, build bodies whose
features sit exactly on those units, and check that the fold reproduces the oracle's bytes."""
import json

import pytest

import _oracle as O

LANE_SPAN = 32
ROUND = 1024
MEMBERS_PER_PASS = 32
MAX_MEMBERS = 128
MAX_PIECES = 96
TEXT_CAP = 3072             # kMutTextCap
COMMA_OFF = TEXT_CAP - 4    # the ',' piece
MAX_KEYS = 16
CLASSES = [(5120, 4), (17408, 2), (65536, 1)]

OK, DECLINED = 0, 4
R_NONE, R_TOO_LARGE, R_SYNTAX, R_ESCAPE, R_TOKENS, R_OPS, R_DUP_KEY, R_UNSUPPORTED, R_ROOT, R_ARENA_FULL = 0, 1, 2, 4, 5, 6, 9, 11, 17, 18
WS = b" \t\r\n"


def mut_class(max_len):
    """(MAXD, warps per CTA) of the launch for a call's max_len (launch_body_mutate)."""
    for maxd, w in CLASSES:
        if max_len <= maxd:
            return maxd, w
    return CLASSES[-1]


def word_copy(l, src, dst):
    """(word path?, head bytes) of one piece: the word path needs l >= 64 and src, dst equal modulo 4."""
    word = l >= 64 and ((src ^ dst) & 3) == 0
    return word, ((4 - (dst & 3)) & 3) if word else 0


# ---------------------------------------------------------------- top-level scan of a JSON object (plain reference of stages A, B)
def scan(body: bytes):
    """Top-level members of a JSON object text: ([(raw key bytes, value start, value end, member start, member end)],
    whitespace outside strings at depth 1?, root open index, root close index).  Member bounds exclude the separators."""
    depth, in_str, esc = 0, False, False
    seps, ws1 = [], False
    for i, c in enumerate(body):
        if in_str:
            if esc:
                esc = False
            elif c == 0x5C:
                esc = True
            elif c == 0x22:
                in_str = False
            continue
        if c == 0x22:
            in_str = True
        elif c in b"{[":
            if depth == 0:
                seps.append(i)
            depth += 1
        elif c in b"}]":
            depth -= 1
            if depth == 0:
                seps.append(i)
        elif c == 0x2C and depth == 1:
            seps.append(i)
        elif c in WS and depth == 1:
            ws1 = True
    assert depth == 0 and not in_str and len(seps) >= 2 and body[seps[0]] == 0x7B
    members = []
    for a, b in zip(seps, seps[1:]):
        s = a + 1
        p = s
        while p < b and body[p] in WS:
            p += 1
        if p == b:
            continue                                      # `{}` / `{ }`
        assert body[p] == 0x22
        q, e = p + 1, False
        while e or body[q] != 0x22:                       # the key's closing quote, escapes honoured
            e = (not e) and body[q] == 0x5C
            q += 1
        key = body[p + 1:q]
        p = q + 1
        while body[p] in WS:
            p += 1
        assert body[p] == 0x3A
        p += 1
        while body[p] in WS:
            p += 1
        ve = b
        while body[ve - 1] in WS:
            ve -= 1
        members.append((key, p, ve, s, b))
    return members, ws1, seps[0], seps[-1]


def config_keys(removes, sets):
    """fill_mutate_params: one entry per distinct key, sets first in configuration order (a later set of the same key replaces the
    value in place), then keys only removed.  Each: dict(name, raw, remove, set)."""
    keys = []
    def find(n):
        return next((k for k in keys if k["name"] == n), None)
    for path, val in sets:
        k = find(path)
        if k is None:
            k = dict(name=path, raw=None, remove=False, set=False); keys.append(k)
        k["set"] = True
        k["raw"] = val if is_json_value(val) else '"' + val + '"'
    for path in removes:
        k = find(path)
        if k is None:
            k = dict(name=path, raw=None, remove=False, set=False); keys.append(k)
        k["remove"] = True
    return keys


def is_json_value(v):
    """isJSONValue as fill_mutate_params restates it (enough of it for the values these tests use)."""
    v = v.strip(" \t\n\v\f\r")
    if v[:1] == '"' and v[-1:] == '"' and len(v) >= 1:
        return True
    if v in ("0", "true", "false", "null"):
        return True
    if v and (v[0].isdigit() or v[0] in "-+") and all(c.isdigit() or c in ".-+eE" for c in v):
        return True
    return bool(v) and ((v[0] == "{" and v[-1] == "}") or (v[0] == "[" and v[-1] == "]"))


def text_layout(removes, sets):
    """Offsets of every key's name, `"key":value` member and value in the shared-memory config text; None when the call
    refuses the configuration with -2 because the text would pass 3 KiB."""
    keys = config_keys(removes, sets)
    o = 0
    for k in keys:
        raw = k["raw"] or ""
        memb = '"' + k["name"] + '":' + raw
        if o + len(k["name"]) + len(memb) + 8 > TEXT_CAP - 8:
            return None
        k["name_off"] = o
        o += (len(k["name"]) + 3) & ~3
        k["memb_off"], k["memb"] = o, memb.encode()
        k["val_off"], k["val"] = o + len(k["name"]) + 3, raw.encode()
        o += (len(memb) + 3) & ~3
    return keys


def expected_status(body: bytes, removes, sets, max_len):
    """(status, reason) the kernel gives a valid JSON object body: the header's decline list made exact."""
    maxd = mut_class(max_len)[0]
    if len(body) == 0:
        return DECLINED, R_SYNTAX
    if len(body) > maxd:
        return DECLINED, R_TOO_LARGE
    members, ws1, _, _ = scan(body)
    if len(members) > MAX_MEMBERS:
        return DECLINED, R_TOKENS
    if any(b"\\" in k for k, *_ in members):
        return DECLINED, R_ESCAPE
    edited = {p.encode() for p in removes if p} | {p.encode() for p, _ in sets if p}
    names = [k for k, *_ in members]
    if any(names.count(e) > 1 for e in edited):
        return DECLINED, R_DUP_KEY
    if ws1 and any(p.encode() in names for p in removes if p):
        return DECLINED, R_UNSUPPORTED
    return OK, R_NONE


def fold_pieces(body: bytes, removes, sets):
    """Stage C restated: the copy pieces [(from text?, source offset, length)] of an OK body, in output order."""
    keys = text_layout(removes, sets)
    members, _, root_open, root_close = scan(body)
    found = {k["name"].encode() for k in keys} & {m[0] for m in members}
    app = [k for k in keys if k["set"] and (k["name"].encode() not in found or k["remove"])]
    by_name = {k["name"].encode(): k for k in keys}
    seps = [root_open] + [m[4] for m in members]        # the separator in front of member i is seps[i]
    pieces = []
    def put(text, src, l):
        if l:
            pieces.append((text, src, l))
    cur = root_open if app else 0
    alive = 0
    for i, (key, vb, ve, ms, me) in enumerate(members):
        k = by_name.get(key)
        act = 0 if k is None else (1 if k["remove"] else 2)
        if act == 1:
            if cur >= 0:
                put(False, cur, seps[i] + (1 if alive == 0 else 0) - cur); cur = -1
        else:
            if cur < 0:
                if alive:
                    put(True, COMMA_OFF, 1)
                cur = ms
            if act == 2:
                put(False, cur, vb - cur); put(True, k["val_off"], len(k["val"])); cur = ve
            alive += 1
    if not app:
        if cur < 0:
            cur = root_close
        put(False, cur, len(body) - cur)
    else:
        if cur >= 0:
            put(False, cur, root_close - cur)
        before = alive > 0
        for k in app:
            if before:
                put(True, COMMA_OFF, 1)
            put(True, k["memb_off"], len(k["memb"])); before = True
        put(False, root_close, 1)
    return pieces


def assemble(body: bytes, removes, sets):
    keys = text_layout(removes, sets)
    text = bytearray(TEXT_CAP)
    text[COMMA_OFF] = 0x2C
    for k in keys:
        text[k["name_off"]:k["name_off"] + len(k["name"])] = k["name"].encode()
        text[k["memb_off"]:k["memb_off"] + len(k["memb"])] = k["memb"]
    return b"".join(bytes(text[s:s + l]) if t else body[s:s + l] for t, s, l in fold_pieces(body, removes, sets))


def copy_paths(body: bytes, removes, sets):
    """[(length, (src ^ dst) & 3, word?, head)] of every piece: shared-memory sources and output records are 16-aligned, so a
    piece's source and destination modulo 4 are its offsets in the staged body or config text and in the record."""
    out, o = [], 0
    for _t, s, l in fold_pieces(body, removes, sets):
        w, h = word_copy(l, s, o)
        out.append((l, (s ^ o) & 3, w, h))
        o += l
    return out


# ---------------------------------------------------------------- generators
ADV = rb'\",\"model\":\"evil\",\"x\":\"'          # string text that reads as members when a quote or escape carry is lost
PREFIX = b'{"f":"'
TAIL = b'","model":"real"}'
# suffixes that follow the filler string's content: (suffix, index of the marked byte, its byte)
FEATURES = {
    "close_quote": (TAIL, 0, b'"'),
    "depth1_comma": (TAIL, 1, b","),
    "open_quote": (b'","a":"' + ADV + TAIL, 6, b'"'),
    "root_close": (TAIL, len(TAIL) - 1, b"}"),
    "bs_run_odd": (b"\\\\\\\"" + TAIL, 2, b"\\"),       # content \\ \" then the closing quote: the run's last byte escapes a quote
    "bs_run_even": (b"\\\\\\\\" + TAIL, 3, b"\\"),      # content \\ \\ then the closing quote
    "nest_open_brace": (b'","n":{"a":[1,{"b":[]}]}' + TAIL[1:], 6, b"{"),
    "nest_open_bracket": (b'","n":{"a":[1,{"b":[]}]}' + TAIL[1:], 11, b"["),
    "nest_close_bracket": (b'","n":{"a":[1,{"b":[]}]}' + TAIL[1:], 22, b"]"),
    "nest_close_brace": (b'","n":{"a":[1,{"b":[]}]}' + TAIL[1:], 23, b"}"),
}
LANE_TARGETS = [95, 96, 97, 543, 544, 545]                    # = 31, 32, 33 (mod 32)
ROUND_TARGETS = [1023, 1024, 1025, 2047, 2048, 2049, 4095, 4096, 4097]   # = 1023, 1024, 1025 (mod 1024)
BIG_TARGETS = [9215, 9216, 9217]                              # inside the 17408 class
ADV_MUTS = [(["model"], []), ([], [("model", '"gpt-x"')]), (["f"], [("z", "1")]), (["x"], [("model", '"m"'), ("x", "2")]), (["n", "a"], [])]


def feature_body(kind, target):
    suffix, idx, ch = FEATURES[kind]
    pad = target - len(PREFIX) - len(ADV) - idx
    assert pad >= 0
    body = PREFIX + b"x" * pad + ADV + suffix
    return body, target, ch


def adversarial_corpus(targets):
    return [(kind, t) + feature_body(kind, t) for kind in FEATURES for t in targets]


RUNS = [1, 2, 3, 31, 32, 33, 63, 64, 65, 1023, 1024, 1025, 2047, 2048, 2049]


def run_body(n, where, in_key=False):
    """A backslash run of n bytes in a value (or a top-level key).  An odd run escapes the quote after it, an even one ends
    before the closing quote.  `where`: ("end", t) puts the run's last byte at t, ("start", t) its first byte."""
    run = b"\\" * n + (b'"q' if n % 2 else b"")
    head = b'{"k' if in_key else b'{"a":"'
    kind, t = where
    first = t if kind == "start" else t - n + 1
    pad = first - len(head)
    assert pad >= 0
    body = head + b"y" * pad + run + (b'":1,"model":"m"}' if in_key else b'","model":"m"}')
    return body, first, first + n - 1


def run_positions(n):
    """end on the last byte of a lane and of a round; start on the first byte of a lane and of a round"""
    pos = [("end", 96 * 32 + 31 if n > 64 else 95), ("end", 2047 + ROUND * ((n + 1023) // 1024)), ("start", 256), ("start", 2048)]
    return pos


def runs_corpus(in_key=False):
    out = []
    for n in RUNS:
        for w in run_positions(n):
            body, a, b = run_body(n, w, in_key)
            out.append((n, w, a, b, body))
    return out


def members_body(n, edited_at=(), key="e", dup_plain=False):
    """n compact members; `key` at every index of edited_at; optionally a non-edited key twice"""
    ms = []
    for i in range(n):
        if i in edited_at:
            ms.append('"%s":"v%d"' % (key, i))
        else:
            ms.append('"m%03d":%d' % (i, i))
    if dup_plain and n >= 4:
        ms[3] = '"m001":3'
    return ("{" + ",".join(ms) + "}").encode()


MEMBER_COUNTS = [1, 31, 32, 33, 64, 127, 128, 129]
EDIT_AT = [0, 31, 32, 63, 64, 127]
MEMBER_MUTS = [(["e"], []), ([], [("e", '"w"')]), (["e"], [("e", "7")]), ([], [("new", "1")]), (["m001"], [])]


def members_corpus():
    out = []
    for n in MEMBER_COUNTS:
        out.append(("count", n, members_body(n)))
        for i in EDIT_AT:
            if i < n:
                out.append(("edit_at_%d" % i, n, members_body(n, (i,))))
    out.append(("dup_in_pass", 40, members_body(40, (3, 20))))
    out.append(("dup_across_passes", 64, members_body(64, (5, 40))))
    out.append(("dup_plain", 40, members_body(40, dup_plain=True)))
    return out


def worst_pieces():
    """16 keys each removed and set, alternating with kept members, every one re-appended: the most pieces a config allows"""
    keys = ["k%02d" % i for i in range(MAX_KEYS)]
    body = ("{" + ",".join('"a%02d":%d,"%s":%d' % (i, i, k, i) for i, k in enumerate(keys)) + ',"z":0}').encode()
    cfgs = [(keys, [(k, str(i)) for i, k in enumerate(keys)]),
            (keys[::2], [(k, '"s%d"' % i) for i, k in enumerate(keys[1::4])] + [("n%02d" % i, "1") for i in range(4)])]
    return body, cfgs


def text_limit_value():
    """the longest JSON string value for a config of two keys ("a" removed, "big" set) that fits the 3 KiB text"""
    n = 2
    while text_layout(["a"], [("big", '"' + "v" * (n + 1 - 2) + '"')]) is not None:
        n += 1
    return '"' + "v" * (n - 2) + '"'


def copy_corpus():
    """kept runs, replacement values and appended members of 63, 64 and 65 bytes.  A deleted member of 1-8 value bytes moves an
    input run's source against its destination; a kept member of 0-3 value bytes in front moves the destination; the key's
    length moves a replacement value's source in the config text (appended members start 4-aligned there)."""
    out = []
    for L in (63, 64, 65):
        for pp in range(4):
            pv = "p" * pp
            keep = '"k":"%s"}' % ("k" * (L - 7))                      # one input piece of L bytes after the deleted member
            for d in range(1, 9):
                out.append(("kept", d, L, ('{"p":"%s","x":"%s",%s' % (pv, "d" * d, keep)).encode(), ["x"], []))
            val = '"' + "r" * (L - 2) + '"'
            for name in ("q", "kk", "kkk", "kkkk"):
                out.append(("value", pp, L, ('{"x":"d","p":"%s","%s":0}' % (pv, name)).encode(), ["x"], [(name, val)]))
            mval = '"' + "m" * (L - 9) + '"'                            # `"apnd":` is 7 bytes
            out.append(("append", pp, L, ('{"x":"d","p":"%s"}' % pv).encode(), ["x"], [("apnd", mval)]))
            out.append(("append", pp, L, ('{"p":"%s"}' % pv).encode(), [], [("apnd", mval)]))
    return out


FLAG_CASES = [  # (body, removes, sets): edits whose record is the input byte for byte, and near misses
    (b'{"a":1}', [], [("a", "1")]),
    (b'{"a":1,"b":2}', [], [("a", "1")]),
    (b'{"b":2,"a":1}', ["a"], [("a", "1")]),
    (b'{"b":2,"a":"s"}', ["a"], [("a", "s")]),
    (b'{"a":1}', [], [("a", "2")]),
    (b'{"a":1,"b":2}', ["a"], [("a", "1")]),
    (b'{"b":2,"a":1}', ["zz"], [("a", "1")]),
    (b'{"a":"xyz"}', [], [("a", "xyz")]),
    (b'{"a":"xyz"}', [], [("a", "xyy")]),
]


def exact_len_body(n):
    """a compact body of exactly n bytes: {"model":"m","pad":"xxx…","t":1}"""
    base = len(b'{"model":"m","pad":"","t":1}')
    return b'{"model":"m","pad":"' + b"x" * (n - base) + b'","t":1}'


CLASS_LENS = [5120, 5121, 17408, 17409, 65536, 65537]


# ---------------------------------------------------------------- self-tests
def _oracle_ok(body, rm, st):
    rc, out = O.body_mutate(body, rm, st)
    assert rc == 0
    return out


def test_constants_and_rules():
    assert [mut_class(m) for m in (1, 5120, 5121, 17408, 17409, 65536, 70000)] == [(5120, 4), (5120, 4), (17408, 2), (17408, 2), (65536, 1), (65536, 1), (65536, 1)]
    assert word_copy(63, 0, 0) == (False, 0) and word_copy(64, 0, 0) == (True, 0) and word_copy(64, 5, 1) == (True, 3)
    assert word_copy(64, 6, 1) == (False, 0) and word_copy(65, 3, 7) == (True, 1) and word_copy(100, 2, 6) == (True, 2)
    assert expected_status(b'{"a":1, "b":2}', ["a"], [], 100) == (DECLINED, R_UNSUPPORTED)
    assert expected_status(b'{"a":1, "b":2}', [], [("a", "5")], 100) == (OK, R_NONE)
    assert expected_status(b'{"a":1,"a":2}', ["a"], [], 100) == (DECLINED, R_DUP_KEY)
    assert expected_status(b'{"a":1,"a":2}', ["b"], [], 100) == (OK, R_NONE)
    assert expected_status(b'{"\\u0061":1}', [], [], 100) == (DECLINED, R_ESCAPE)
    assert expected_status(b'{"a":{"b" : 1}}', ["a"], [], 100) == (OK, R_NONE)       # whitespace at depth 2 is no matter
    assert expected_status(b" " * 5121, [], [], 5120) == (DECLINED, R_TOO_LARGE)
    assert expected_status(exact_len_body(5121), [], [], 5121) == (OK, R_NONE)


def test_fold_reproduces_the_oracle():
    """the restated piece fold gives the oracle's bytes for every OK body of every corpus here"""
    cases = [(b, rm, st) for _k, _t, b, _o, _c in adversarial_corpus(LANE_TARGETS[:3] + ROUND_TARGETS[:3]) for rm, st in ADV_MUTS]
    cases += [(b, rm, st) for _k, _n, b in members_corpus() for rm, st in MEMBER_MUTS]
    cases += [(b, rm, st) for _k, _d, _L, b, rm, st in copy_corpus()]
    cases += FLAG_CASES
    body, cfgs = worst_pieces()
    cases += [(body, rm, st) for rm, st in cfgs]
    n_ok = 0
    for b, rm, st in cases:
        if expected_status(b, rm, st, 65536)[0] == OK:
            assert assemble(b, rm, st) == _oracle_ok(b, rm, st), (b[:120], rm, st)
            n_ok += 1
    assert n_ok > 500


@pytest.mark.parametrize("targets", [LANE_TARGETS, ROUND_TARGETS, BIG_TARGETS])
def test_adversarial_features_land_on_their_targets(targets):
    corpus = adversarial_corpus(targets)
    assert {k for k, *_ in corpus} == set(FEATURES) and len(corpus) == len(FEATURES) * len(targets)
    for kind, t, body, off, ch in corpus:
        json.loads(body)
        assert off == t and body[off:off + 1] == ch, (kind, t)
        assert ADV in body and json.loads(body)["model"] == "real"
        members, ws1, _, _ = scan(body)
        assert not ws1 and [m[0] for m in members][-1] == b"model" and len(members) in (2, 3)
    mods = {t % LANE_SPAN for t in targets} | {t % ROUND for t in targets}
    assert {31, 0, 1} <= mods or {1023, 0, 1} <= mods


def test_backslash_runs_cover_lanes_and_rounds():
    for in_key in (False, True):
        seen_end_lane = seen_end_round = seen_start_lane = seen_start_round = seen_full_lane = seen_full_round = 0
        for n, w, a, b, body in runs_corpus(in_key):
            d = json.loads(body)
            assert body[a:b + 1] == b"\\" * n and body[a - 1] != 0x5C and body[b + 1] == 0x22
            key = scan(body)[0][0][0]
            if in_key:
                assert b"\\" in key and expected_status(body, [], [], 65536) == (DECLINED, R_ESCAPE)
            else:
                assert d["a"].endswith("\\" * (n // 2) + ('"q' if n % 2 else "")) and expected_status(body, ["model"], [], 65536) == (OK, R_NONE)
            seen_end_lane += b % 32 == 31
            seen_end_round += b % 1024 == 1023
            seen_start_lane += a % 32 == 0
            seen_start_round += a % 1024 == 0
            seen_full_lane += (b + 1) // 32 - (a + 31) // 32 >= 1        # a whole lane of backslashes: the `full` mask
            seen_full_round += (b + 1) // 1024 - (a + 1023) // 1024 >= 1
        assert min(seen_end_lane, seen_end_round, seen_start_lane, seen_start_round) >= len(RUNS)
        assert seen_full_lane >= 20 and seen_full_round >= 8
    assert {n % 2 for n in RUNS} == {0, 1}


def test_member_counts_and_edit_positions():
    corpus = members_corpus()
    for kind, n, body in corpus:
        members = scan(body)[0]
        assert len(members) == n
        if kind.startswith("edit_at_"):
            assert members[int(kind[8:])][0] == b"e"
    st = {(k, n): expected_status(b, ["e"], [], 65536) for k, n, b in corpus}
    assert st[("count", 128)] == (OK, R_NONE) and st[("count", 129)] == (DECLINED, R_TOKENS)
    assert st[("edit_at_127", 128)] == (OK, R_NONE) and st[("edit_at_127", 129)] == (DECLINED, R_TOKENS)
    assert st[("dup_in_pass", 40)] == (DECLINED, R_DUP_KEY) and st[("dup_across_passes", 64)] == (DECLINED, R_DUP_KEY)
    assert st[("dup_plain", 40)] == (OK, R_NONE)
    dups = {k: [i for i, m in enumerate(scan(b)[0]) if m[0] == b"e"] for k, _n, b in corpus if k.startswith("dup_")}
    assert dups["dup_in_pass"] == [3, 20] and dups["dup_across_passes"] == [5, 40]
    assert dups["dup_across_passes"][0] // MEMBERS_PER_PASS != dups["dup_across_passes"][1] // MEMBERS_PER_PASS


def test_piece_cap_is_unreachable():
    body, cfgs = worst_pieces()
    counts = []
    for rm, st in cfgs:
        assert len(config_keys(rm, st)) == MAX_KEYS
        assert expected_status(body, rm, st, 65536) == (OK, R_NONE)
        counts.append(len(fold_pieces(body, rm, st)))
    assert counts == [66, 34]
    # every edited member adds at most 2 pieces, every appended key 2, the last run and the closing brace 2: 16 * 2 + 16 * 2 + 2
    assert 2 * MAX_KEYS + 2 * MAX_KEYS + 2 < MAX_PIECES


def test_text_limit():
    v = text_limit_value()
    assert text_layout(["a"], [("big", v)]) is not None
    assert text_layout(["a"], [("big", v[:-1] + 'v"')]) is None
    assert 3000 < len(v) < TEXT_CAP


def test_copy_paths_cover_every_alignment():
    word_heads, byte_mis, lens = set(), set(), set()
    for kind, d, L, body, rm, st in copy_corpus():
        assert expected_status(body, rm, st, 65536) == (OK, R_NONE)
        ps = copy_paths(body, rm, st)
        assert any(l == L for l, *_ in ps), (kind, d, L)
        for l, mis, w, h in ps:
            if l >= 64 and w:
                word_heads.add((kind.split("_")[0], h))
            if l >= 64 and not w:
                byte_mis.add((kind.split("_")[0], mis))
            lens.add(l)
    for kind in ("kept", "value", "append"):
        assert {h for k, h in word_heads if k == kind} == ({0} if kind == "append" else {0, 1, 2, 3}), kind
        assert {m for k, m in byte_mis if k == kind} == {1, 2, 3}, kind
    assert {63, 64, 65} <= lens


def test_flag_cases_and_class_bodies():
    same = [assemble(b, rm, st) == b for b, rm, st in FLAG_CASES]
    assert same == [True, True, True, True, False, False, True, True, False]
    for n in CLASS_LENS:
        b = exact_len_body(n)
        assert len(b) == n and json.loads(b)["model"] == "m"
