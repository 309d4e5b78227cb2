"""Generators for the SSE usage scan edge tests (test_sse_usage_edges_gpu.py) and their self-checks (no GPU).

sse_usage_kernel (aigw_b200/csrc/sse_kernel.cu) scans one stream per warp in fixed units:
  tile       up to 8192 bytes: the unterminated line the previous tile left (the carry) plus the next bytes of the stream,
             staged at t0 = (address of the tile's first byte) mod 16
  chunk      16 bytes of the tile per lane, 512 bytes per group of 32 lanes.  Newlines, `"usage"` and `\\u` are found per chunk;
             the `u` after a `"` or `\\` in the chunk's last byte is read from the next chunk (`next_u`)
  lines      at most 512 newlines per tile, else the stream declines; a tile that fills to 8192 bytes without a newline declines
  candidates at most 64 listed per tile; past 64 every line of the tile is decoded.  The tile's last two `data: ` lines are
             always decoded; when neither yields a model, every line of the tile is decoded again (the walk-all pass)
  carry      the tail after the tile's last newline moves to tile[nt0], nt0 = its address mod 16
The helpers restate that schedule in plain Python and build streams that sit exactly on those numbers."""
import json

import pytest

import _oracle as O

TILE = 8192
CHUNK = 16
GROUP = 512
MAX_LINES = 512
MAX_CAND = 64
DATA = b"data: "


def candidates(tile: bytes, lo: int, hi: int):
    """tile indices of `"usage"` and `\\u` candidates in tile[lo:hi], as the kernel finds them (a `u` at tile[hi] is stale data
    of an earlier tile for the kernel: a `\\` in the last staged byte may or may not count, and never changes which line is
    decoded, so it is left out here)"""
    out = []
    for j in range(lo, hi):
        c = tile[j]
        if c not in b'"\\' or j + 1 >= hi or tile[j + 1] != 0x75:
            continue
        if c == 0x22 and not (j + 6 < hi and tile[j + 2:j + 7] == b'sage"'):
            continue
        out.append(j)
    return out


def tile_schedule(stream: bytes, start_mod16: int):
    """([(tile_base, t0, filled, nlines, ncand, cand1, cand2, carry_move, cand_positions)], declined).  tile_base is the stream
    offset of the tile's first data byte; cand1 / cand2 are line indices (None when absent); carry_move is 'none', 'down' or
    'up'; cand_positions are tile indices."""
    n = len(stream)
    pos, carry, t0 = 0, 0, start_mod16 & 15
    tiles = []
    while pos < n or carry:
        take = min(TILE - carry, n - pos)
        if take == 0 and pos >= n:
            break
        filled = carry + take
        base = pos - carry
        pos += take
        data = stream[base:base + filled]
        tile = b"\0" * t0 + data
        nl = [t0 + i for i, c in enumerate(data) if c == 0x0A]
        cands = candidates(tile, t0, t0 + filled)
        if not nl:
            if filled >= TILE:
                return tiles, True
            if pos >= n:
                break
            carry = filled
            continue
        if len(nl) > MAX_LINES:
            return tiles, True
        data_lines = []
        for li, e in enumerate(nl):
            b = t0 if li == 0 else nl[li - 1] + 1
            if e - b >= 6 and tile[b:b + 6] == DATA:
                data_lines.append(li)
        cand1 = data_lines[-1] if data_lines else None
        cand2 = data_lines[-2] if len(data_lines) > 1 else None
        last = nl[-1] + 1
        rem = t0 + filled - last
        nt0 = (start_mod16 + pos - rem) & 15
        move = "none" if rem == 0 or nt0 == last else ("down" if nt0 < last else "up")
        tiles.append((base, t0, filled, len(nl), len(cands), cand1, cand2, move, cands))
        t0, carry = nt0, rem
        if pos >= n:
            break
    return tiles, False


def expected_declined(stream: bytes):
    """the stream declines exactly when a tile has more than 512 newlines or fills to 8192 bytes without one (an unterminated tail
    of 8192 bytes or more included); independent of the start address.  Holds for streams whose decoded lines never set `weird`."""
    return tile_schedule(stream, 0)[1]


# ---------------------------------------------------------------- line shapes the kernel decodes
def chunk(model, content="x", usage=None):
    d = {"id": "c", "object": "chat.completion.chunk", "created": 1, "model": model, "choices": [{"index": 0, "delta": {"content": content}}]}
    if usage is not None:
        d["usage"] = usage
    return ("data: " + json.dumps(d, separators=(",", ":")) + "\n\n").encode()


def U(a, b, cached=None):
    u = {"prompt_tokens": a, "completion_tokens": b, "total_tokens": a + b}
    if cached is not None:
        u["prompt_tokens_details"] = {"cached_tokens": cached}
    return u


DONE, COMMENT, PING, BROKEN = b"data: [DONE]\n\n", b": comment\n\n", b"event: ping\n\n", b"data: {oops\n\n"


def comment_line(L):
    """a line of exactly L bytes with its newline"""
    return b"\n" if L == 1 else b":\n" if L == 2 else b": " + b"c" * (L - 3) + b"\n"


def fill_lines(nbytes, nlines):
    """nlines lines of nbytes bytes in all"""
    base, extra = divmod(nbytes, nlines)
    assert base >= 1
    return b"".join(comment_line(base + (i < extra)) for i in range(nlines))


def pad_to(prefix: bytes, addr_mod: int, modulus: int, start_mod16: int, marker: bytes, line_fn):
    """line_fn(k) -> a line with `marker`; pick k so that marker's first byte sits at an address = addr_mod (mod modulus), the
    stream starting at an address = start_mod16 (mod 16, and 0 mod modulus otherwise)"""
    for k in range(modulus + 1):
        ln = line_fn(k)
        a = start_mod16 + len(prefix) + ln.index(marker)
        if a % modulus == addr_mod:
            return ln
    raise AssertionError("no padding")


# ---------------------------------------------------------------- streams
def s_next_u(start, marker=b'"usage"', modulus=CHUNK, addr=15):
    """a usage line whose `"usage"` quote sits at address = addr (mod modulus) and is not one of its tile's last two data lines:
    only `next_u` (for addr = 15 mod 16) lists it.  The last two data lines carry a model, so the walk-all pass does not run."""
    pre = chunk("m0") + COMMENT
    ln = pad_to(pre, addr, modulus, start, marker, lambda k: chunk("m0", content="t" * k, usage=U(11, 22, 3)))
    return pre + ln + chunk("m1") + chunk("m2", content="é") + PING


def s_second_pass(start):
    """the model sits before the tile's last two data lines, which decode with an empty model or not at all"""
    return [chunk("M1") + chunk("") + BROKEN + COMMENT,
            chunk("A", usage=U(1, 2)) + chunk("B") + chunk("") + DONE,
            chunk("only") + BROKEN + BROKEN,
            chunk("early") + COMMENT * 3 + chunk("", usage=U(4, 5)) + chunk("")]


def s_model_across_tiles():
    """the last model-bearing line is in an earlier tile: later tiles hold comments, broken lines and empty models"""
    tail = (BROKEN + COMMENT + chunk("") + PING) * 200
    return chunk("carried", usage=U(7, 8)) + tail, chunk("first") + tail + chunk("", usage=U(9, 9)) + tail


def s_lines_per_tile(nl, start_lines=b""):
    """a first tile of exactly 8192 bytes ending in a newline with `nl` newlines, after a prefix, then usage and model lines"""
    pre = chunk("pre", usage=U(5, 6)) + start_lines
    body = fill_lines(TILE - len(pre), nl - pre.count(b"\n"))
    return pre + body + chunk("post", usage=U(1, 1)) + DONE


def s_long_line(L, terminated=True):
    """a data line of L bytes with its newline (or an unterminated tail of L bytes), after a usage line"""
    pre = chunk("p", usage=U(2, 3))
    ln = chunk("long", content="")
    fill = L - len(ln) + 1                      # ln ends in two newlines: the line itself is len(ln) - 1 bytes
    ln = chunk("long", content="z" * fill)[:-1]
    assert len(ln) == L
    return pre + (ln if terminated else ln[:-1]) + (chunk("after") if terminated else b"")


def s_candidates(k):
    """a first tile whose `"usage"` / `\\u` positions number k: one `\\u` per é of the content"""
    pre = chunk("c0", usage=U(3, 4))           # 1 candidate
    return pre + chunk("c1", content="é" * (k - 1)) + COMMENT * 4 + chunk("c2") + chunk("c3")


def boundary_streams():
    """(name, stream) pairs for every unit edge; each is used at every start offset"""
    out = []
    for nl in (511, 512, 513):
        out.append(("lines_%d" % nl, s_lines_per_tile(nl)))
    for L in (8191, 8192, 8193):
        out.append(("line_%d" % L, s_long_line(L)))
        out.append(("tail_%d" % L, s_long_line(L, terminated=False)))
    for k in (63, 64, 65):
        out.append(("cand_%d" % k, s_candidates(k)))
    a, b = s_model_across_tiles()
    out += [("model_across_a", a), ("model_across_b", b)]
    return out


def usage_split_stream():
    """`"usage"` cut by the end of the first full tile, for every cut inside the key: the line is carried whole"""
    out = []
    ln = chunk("s", content="", usage=U(6, 7))
    k = ln.index(b'"usage"')
    for cut in range(1, 7):
        pre_len = TILE - (k + cut)
        pre = chunk("m") + fill_lines(pre_len - len(chunk("m")), 60)
        out.append(pre + ln + chunk("m2") + DONE)
    return out


def big_stream(mb, seed):
    import random
    r = random.Random(seed)
    parts, n = [], 0
    while n < mb << 20:
        x = r.random()
        p = chunk(r.choice(["a", "b", "gpt-4o", ""]), content="t" * r.randint(0, 400)) if x < 0.7 else \
            chunk(r.choice(["u", "v"]), usage=U(r.randint(0, 999), r.randint(0, 999))) if x < 0.75 else \
            r.choice([DONE, COMMENT, PING, BROKEN, chunk("e", content="é" * r.randint(1, 5))])
        parts.append(p); n += len(p)
    return b"".join(parts)


# ---------------------------------------------------------------- self-tests
def _sched(s, start=0):
    return tile_schedule(s, start)


def test_schedule_known_answers():
    s = chunk("a") + COMMENT
    tiles, d = _sched(s, 3)
    assert not d and len(tiles) == 1 and tiles[0][:4] == (0, 3, len(s), 4)
    assert _sched(b"x" * 8191, 0) == ([], False)                # an unterminated tail under 8192 bytes is never parsed
    assert _sched(b"x" * 8192, 0)[1] and _sched(b"x" * 9000, 0)[1]
    assert not _sched(b"x" * 8191 + b"\n", 0)[1] and _sched(b"x" * 8192 + b"\n", 0)[1]
    assert candidates(b'x"usage"', 0, 8) == [1] and candidates(b'x"usage', 0, 7) == [] and candidates(b"\\u00", 0, 4) == [0]


def test_boundary_streams_hit_their_edges():
    bs = dict(boundary_streams())
    for nl in (511, 512, 513):
        tiles, d = _sched(bs["lines_%d" % nl])
        assert d == (nl > MAX_LINES)
        if not d:
            assert tiles[0][2] == TILE and tiles[0][3] == nl
    for L in (8191, 8192, 8193):
        s = bs["line_%d" % L]
        lines = s.split(b"\n")
        assert max(len(x) for x in lines) + 1 == L
        assert expected_declined(s) == (L > TILE)
        t = bs["tail_%d" % L]
        assert not t.endswith(b"\n") and len(t) - t.rindex(b"\n") - 1 == L - 1
        assert expected_declined(t) == (len(t) - t.rindex(b"\n") - 1 >= TILE)
    assert [expected_declined(bs["tail_%d" % L]) for L in (8191, 8192, 8193)] == [False, False, True]
    assert [expected_declined(bs["line_%d" % L]) for L in (8191, 8192, 8193)] == [False, False, True]
    for k in (63, 64, 65):
        tiles, d = _sched(bs["cand_%d" % k])
        assert not d and tiles[0][4] == k
    for name in ("model_across_a", "model_across_b"):
        tiles, d = _sched(bs[name])
        assert not d and len(tiles) >= 3


def test_start_offsets_and_chunk_edges():
    seen15_q = seen15_bs = g511 = g0 = 0
    for start in range(16):
        s = s_next_u(start)
        tiles, d = _sched(s, start)
        assert not d and len(tiles) == 1
        t0 = tiles[0][1]
        assert t0 == start
        q = s.index(b'"usage"')
        assert (start + q) % CHUNK == 15 and (t0 + q) in tiles[0][8]
        # the usage line is neither of the tile's last two data lines
        line_of_q = s[:q].count(b"\n")
        assert line_of_q not in (tiles[0][5], tiles[0][6])
        seen15_q += 1
        for tb, t0_, filled, nl, nc, c1, c2, mv, cands in tiles:
            seen15_bs += sum(1 for c in cands if c % CHUNK == 15)
        s2 = s_next_u(start, marker=b'"usage"', modulus=GROUP, addr=511)
        q2 = s2.index(b'"usage"')
        assert (start + q2) % GROUP == 511
        g511 += 1
        s3 = s_next_u(start, marker=b'"usage"', modulus=GROUP, addr=0)
        g0 += (start + s3.index(b'"usage"')) % GROUP == 0
    assert seen15_q == 16 and g511 == 16 and g0 == 16 and seen15_bs >= 16


def test_split_usage_is_carried():
    for s in usage_split_stream():
        tiles, d = _sched(s)
        assert not d and len(tiles) >= 2
        q = s.index(b'"usage"')
        assert tiles[0][2] == TILE and q < TILE < q + 7       # the key straddles the first tile's end
        assert all(tiles[0][0] + c - tiles[0][1] != q for c in tiles[0][8])
        assert any(tiles[1][0] + c - tiles[1][1] == q for c in tiles[1][8])


def test_carry_never_moves_up():
    """the tail keeps its address modulo 16, so its new start nt0 = last mod 16 <= last: the carry moves down or stays, and
    when the tile's last newline lies in its first 16 bytes it stays where it is"""
    moves = set()
    stay_first16 = 0
    for start in range(16):
        for s in [s_next_u(start)] + [x for _n, x in boundary_streams()][:6] + [COMMENT + b"x" * 9000, b"\n" + b"y" * 8000 + b"\nq"]:
            tiles, _ = _sched(s, start)
            for tb, t0, filled, nl, nc, c1, c2, mv, cands in tiles:
                moves.add(mv)
    for start in range(16):
        s = b"\n" + b"y" * 9000 + b"\n"
        tiles, _ = _sched(s, start)
        stay_first16 += tiles[0][7] == "none" and tiles[0][3] == 1
    # the newline sits at tile[start]: the tail starts at start + 1, inside the first 16 bytes for starts 0-14, and stays there
    assert "up" not in moves and {"down", "none"} <= moves and stay_first16 == 15


def test_second_pass_and_carried_models_need_them():
    for s in s_second_pass(0):
        tiles, d = _sched(s)
        assert not d and len(tiles) == 1
        st = O.SSEStream(); st.feed(s)
        model = st.model()
        c1, c2 = tiles[0][5], tiles[0][6]
        lines = s.split(b"\n")
        # the model line is an earlier line than both candidates
        idx = next(i for i, ln in enumerate(lines) if b'"model":"%s"' % model in ln)
        assert model and idx < min(x for x in (c1, c2) if x is not None)
    a, b = s_model_across_tiles()
    for s, m in ((a, b"carried"), (b, b"first")):
        st = O.SSEStream(); st.feed(s)
        assert st.model() == m
        tiles, _ = _sched(s)
        assert s.index(b'"model":"%s"' % m) < tiles[1][0]


def test_big_streams_have_hundreds_of_tiles():
    for mb, seed in ((1, 1), (4, 2)):
        s = big_stream(mb, seed)
        tiles, d = _sched(s, 5)
        assert not d and len(tiles) >= 120 * mb
