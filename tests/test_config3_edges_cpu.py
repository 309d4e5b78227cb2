"""Generators for the config-3 edge tests (test_config3_edges_gpu.py) and their self-checks (no GPU).

BASELINE config 3 runs emb_scan_kernel -> bpe_count_kernel -> emb_sum_kernel.  Both kernels work in fixed units:
  bpe_count_kernel  a warp stages groups of up to 32 consecutive texts into a 512-byte buffer; a longer text is cut at piece
                    boundaries, and a text with a piece longer than the buffer is declined (0xFFFFFFFF); the merge table is an
                    open-addressing hash in shared memory (bpe_hash, linear probing that wraps from slot `mask` to 0)
  emb_scan_kernel   a CTA of 256 threads streams a request in 8192-byte tiles, 32 bytes per thread, so thread boundaries fall every
                    32 bytes, warp boundaries every 1024 and tile boundaries every 8192
The helpers here restate the decline rule and the table layout in plain Python and build texts, vocabularies and request bodies
that sit exactly on those numbers."""
import json

import numpy as np
import pytest

import _oracle as O

BUF = 512                   # bpe_count_kernel's staging buffer (kBpeBuf)
GROUP = 32                  # texts per group (kBpeMaxTexts)
TILE = 8192                 # emb_scan_kernel: 256 threads x 32 bytes
WARP_SPAN = 1024
THREAD_SPAN = 32
DECLINED = 0xFFFFFFFF
MAX_ID = 65534              # aigw_bpe_load refuses ids of 65535 and above


# ---------------------------------------------------------------- pre-tokenisation and the decline rule
def pieces(text: bytes):
    """Every space starts a new piece; a piece is its first byte plus the bytes up to the next space (the text's first byte
    starts a piece whether or not it is a space)."""
    out, i, n = [], 0, len(text)
    while i < n:
        j = i + 1
        while j < n and text[j] != 0x20:
            j += 1
        out.append(text[i:j])
        i = j
    return out


def declined(text: bytes) -> bool:
    """aigw_bpe_count_*: a text is declined exactly when one of its pieces is longer than the 512-byte staging buffer."""
    return any(len(p) > BUF for p in pieces(text))


def test_pieces_known_answers():
    assert pieces(b"") == []
    assert pieces(b"a") == [b"a"]
    assert pieces(b"ab cd") == [b"ab", b" cd"]
    assert pieces(b" ab") == [b" ab"]
    assert pieces(b"  ab ") == [b" ", b" ab", b" "]
    assert pieces(b"   ") == [b" ", b" ", b" "]
    assert pieces(b"\x00 \xff") == [b"\x00", b" \xff"]


@pytest.mark.parametrize("text,want", [
    (b"", False), (b"x" * 512, False), (b"x" * 513, True),
    (b"x" * 512 + b" y", False), (b"x" * 513 + b" y", True),           # the first piece has no leading space
    (b"y " + b"x" * 511, False), (b"y " + b"x" * 512, True),           # a later piece counts its space: 1 + 511 = 512 fits
    (b"y " + b"x" * 511 + b" z", False), (b"y " + b"x" * 512 + b" z", True),
    (b" " * 600, False), (b"a " * 300, False), (b" " + b"x" * 511, False), (b" " + b"x" * 512, True),
    (b"x" * 1000 + b" " + b"y" * 10, True), (b"y" * 10 + b" " + b"x" * 511 + b" " + b"z" * 511, False),
], ids=lambda v: f"{len(v)}B" if isinstance(v, bytes) else str(v))
def test_decline_rule_known_answers(text, want):
    assert declined(text) is want


# ---------------------------------------------------------------- the merge table (aigw_bpe_load, bpe_kernel.cu)
def bpe_hash(key: int) -> int:
    """bpe_hash: key * 0x9E3779B1 (mod 2^32), then xor with itself shifted right by 15."""
    key = (key * 0x9E3779B1) & 0xFFFFFFFF
    return key ^ (key >> 15)


def slots_for(n_merges: int) -> int:
    """aigw_bpe_load: at least 1024 slots, the smallest power of two holding two slots per merge."""
    s = 1024
    while s < n_merges * 2:
        s <<= 1
    return s


def fits_shared_memory(n_merges: int) -> bool:
    """bpe_smem_bytes(slots) <= 220 KiB: 8 bytes per slot plus 32 warps' staging buffers (sizeof(BpeWarpSmem) = 3932)."""
    return slots_for(n_merges) * 8 + 32 * 3932 <= 220 * 1024


def home(a: int, b: int, slots: int) -> int:
    return bpe_hash((a << 16) | b) & (slots - 1)


def table_layout(merges, slots):
    """Where aigw_bpe_load puts each pair: {key: slot}; a repeated pair keeps its first slot (and rank)."""
    mask = slots - 1
    tab, where = {}, {}
    for a, b, _ in merges:
        key = (a << 16) | b
        if key in where:
            continue
        s = bpe_hash(key) & mask
        while s in tab:
            s = (s + 1) & mask
        tab[s] = key
        where[key] = s
    return where


def identity_b2i():
    return list(range(256))


def collision_vocab():
    """Pairs of byte ids whose home slots are mask-2, mask-1 and mask of a 1024-slot table, three per home, so that the probe runs
    through slot `mask` and wraps around to 0, 1, 2, ...; every pair merges into a fresh id, and a few second-level merges make the
    merged ids meet again.  Returns (vocab dict, the colliding pairs)."""
    slots = 1024
    mask = slots - 1
    letters = list(range(0x21, 0x7F))
    want = {mask - 2: [], mask - 1: [], mask: []}
    for a in letters:
        for b in letters:
            h = home(a, b, slots)
            if h in want and len(want[h]) < 3 and a not in (0x22, 0x5C) and b not in (0x22, 0x5C):
                want[h].append((a, b))
    pairs = want[mask - 2] + want[mask - 1] + want[mask]
    assert len(pairs) == 9
    merges, nid = [], 256
    ids = {}
    for a, b in pairs:
        merges.append((a, b, nid)); ids[(a, b)] = nid; nid += 1
    # second level: the merged id of pair k followed by the first byte of pair k + 1
    for k in range(len(pairs) - 1):
        merges.append((ids[pairs[k]], pairs[k + 1][0], nid)); nid += 1
    return {"byte_to_id": identity_b2i(), "merges": [list(m) for m in merges]}, pairs


def chain_vocab_binary(depth: int):
    """'a' -> aa -> a4 -> ... -> a(2^depth): merge (a_k, a_k) -> a_2k with rank k.  tokens('a' * n) = (n >> depth) + popcount(n mod 2^depth)."""
    a = ord("a")
    merges, cur = [], a
    for k in range(depth):
        merges.append((cur, cur, 256 + k)); cur = 256 + k
    return {"byte_to_id": identity_b2i(), "merges": [list(m) for m in merges]}


def chain_vocab_linear(k: int):
    """t_i + 'a' -> t_(i+1) ranked before 'a' + 'a' -> t_2, up to t_k: on 'a' * n the leftmost token grows to k bytes before the
    next one starts, so tokens('a' * n) = ceil(n / k)."""
    a = ord("a")
    merges = [(256 + i - 2, a, 256 + i - 1) for i in range(2, k)]   # t_i has id 256 + i - 2 (t_2 = 256)
    merges.append((a, a, 256))
    return {"byte_to_id": identity_b2i(), "merges": [list(m) for m in merges]}


def largest_vocab(n_merges: int):
    """n_merges distinct pairs of printable bytes, each merging into a fresh id (ranks in order)."""
    letters = [c for c in range(0x21, 0x7F) if c not in (0x22, 0x5C)]
    merges = []
    for i in range(n_merges):
        a, b = letters[i % len(letters)], letters[(i // len(letters)) % len(letters)]
        merges.append((a, b, 256 + i))
    return {"byte_to_id": identity_b2i(), "merges": [list(m) for m in merges]}


def high_id_vocab():
    """A non-identity byte_to_id (bytes 'a'..'z' fold onto 13 ids near the top of the range, other bytes keep their value) and merged
    ids up to 65534, the largest id aigw_bpe_load accepts."""
    b2i = identity_b2i()
    for c in range(ord("a"), ord("z") + 1):
        b2i[c] = MAX_ID - 20 - (c - ord("a")) % 13                        # a and n share an id, b and o, ...
    x = lambda ch: b2i[ord(ch)]
    merges = [(x("a"), x("b"), MAX_ID), (MAX_ID, x("c"), MAX_ID - 1), (x("d"), x("e"), MAX_ID - 2), (MAX_ID - 2, MAX_ID - 1, MAX_ID - 3),
              (MAX_ID, MAX_ID, MAX_ID - 4), (ord(" "), MAX_ID, MAX_ID - 5), (x("z"), x("z"), MAX_ID - 6)]
    return {"byte_to_id": b2i, "merges": [list(m) for m in merges]}


def duplicate_vocab():
    """(a, b) appears at rank 0 -> X and again at rank 3 -> Y; only X merges on with c, so the first rank is observable."""
    a, b, c = ord("a"), ord("b"), ord("c")
    merges = [(a, b, 300), (b, c, 301), (300, c, 302), (a, b, 303), (303, c, 304), (b, b, 305), (b, b, 306)]
    return {"byte_to_id": identity_b2i(), "merges": [list(m) for m in merges]}


# ---------------------------------------------------------------- staging-edge texts
WORDS = b"lorem ipsum dolor sit amet consectetur adipiscing elit sed do eiusmod tempor incididunt ut labore et dolore magna aliqua".split()


def words_text(n: int, seed: int) -> bytes:
    """Exactly n bytes of space-separated words (no piece longer than 12 bytes)."""
    r = np.random.default_rng(seed)
    out = bytearray()
    while len(out) < n:
        if out:
            out += b" "
        out += WORDS[int(r.integers(len(WORDS)))]
    return bytes(out[:n])


def run(n: int, byte=b"x") -> bytes:
    return byte * n


def staging_texts():
    """Texts around the 512-byte staging buffer and the cut rule."""
    t = []
    for n in list(range(0, 80)) + list(range(490, 540)) + [600, 1023, 1024, 1025, 1536, 2048]:
        t.append(words_text(n, n))            # text lengths around 511 / 512 / 513 (all counted: short pieces)
        t.append(run(n))                      # one piece: counted up to 512 bytes, declined above
        t.append(b" " + run(max(0, n - 1)))   # one piece with its leading space
    # multi-run texts whose cuts land at byte 1, 511 and 512 of the window
    for cut in (1, 2, 31, 32, 33, 510, 511, 512):
        head = run(cut, b"h") if cut > 0 else b""
        for tail in (1, 200, 511, 512, 513, 900):
            t.append(head + b" " + run(tail - 1, b"t"))                     # first piece ends at `cut`, then a piece of `tail` bytes
            t.append(head + b" " + run(tail - 1, b"t") + b" end")
    # pieces of 511, 512 and 513 bytes at the start, in the middle and at the end of a text
    for p in (511, 512, 513):
        body = b"y" * (p - 1)
        t.append(b"x" + body + b" mid dle")                                 # first piece: p bytes without a space
        t.append(b"pre fix " + b"z" * (p - 1) + b" post")                    # a middle piece: space + p - 1 bytes = p
        t.append(b"pre fix" + b" " + b"z" * (p - 1))                         # last piece
        t.append(words_text(700, p) + b" " + b"w" * (p - 1) + b" " + words_text(700, p + 1))
    # spaces: runs, only spaces, leading and trailing
    for n in (1, 2, 31, 32, 33, 511, 512, 513, 1100):
        t.append(b" " * n)
        t.append(b" " * n + b"lead")
        t.append(b"trail" + b" " * n)
        t.append(b"a" + b" " * n + b"b" + b"  " + b"c")
    # every byte value, NUL and 0x80..0xFF included, alone, in pairs and in one long text
    t += [bytes([v]) for v in range(256)]
    t += [bytes([v, (v * 7 + 3) & 0xFF, v]) for v in range(256)]
    t.append(bytes(range(256)) * 3)
    t.append(bytes(v for v in range(256) if v != 0x20) * 2)                # 510-byte pieces
    return t


def decline_texts():
    """Texts that are declined only under a rule off by one (or by the buffer's full 512 bytes)."""
    t = []
    for pre in (b"", b"a", b"a b", words_text(300, 1), words_text(511, 2), words_text(512, 3), words_text(513, 4)):
        for p in (510, 511, 512, 513, 514):
            piece = b" " + b"q" * (p - 1)
            t.append(pre + piece)
            t.append(pre + piece + b" r")
            t.append(pre + piece + piece)
            t.append(pre + piece + b" " + words_text(100, p))
    return t


def fill_calls():
    """Calls whose first k texts (one group starts at text 0) fill the 512-byte buffer exactly, or stop one byte short of it or
    one byte past it, followed by a few more texts.  Returns [(total, k, texts)]."""
    calls = []
    for total in (511, 512, 513):
        for k in (1, 2, 3, 8, 31, 32):
            base, extra = divmod(total, k)
            t = [words_text(base + (1 if i < extra else 0), 1000 * total + 10 * k + i) for i in range(k)]
            calls.append((total, k, t + [words_text(n, n) for n in (1, 2, 100, 511, 512)]))
    return calls


def group_calls():
    """Calls of 31, 32, 33, 63, 64 and 65 texts, each with a long text first, last and in the middle, and empty texts between long ones."""
    calls = []
    for n in (31, 32, 33, 63, 64, 65):
        for where in ("first", "middle", "last", "none"):
            texts = [words_text(20 + (i * 37) % 90, 7 * n + i) for i in range(n)]
            at = {"first": 0, "middle": n // 2, "last": n - 1}.get(where)
            if at is not None:
                texts[at] = words_text(1500, n) + b" " + b"k" * 511 + b" " + words_text(700, n + 1)
            calls.append(texts)
        calls.append([b"" if i % 2 else words_text(600 + i, i) for i in range(n)])   # empty texts between long ones
    return calls


def test_generators_sit_on_the_edges():
    st = staging_texts()
    lens = {len(x) for x in st}
    assert {0, 511, 512, 513}.issubset(lens)
    assert any(declined(x) for x in st) and any(not declined(x) and len(x) > BUF for x in st)
    # some text is counted under the fixed rule although a 512-byte window starting at a piece start holds no other space
    assert any(not declined(x) and any(len(p) == BUF for p in pieces(x)[:-1]) for x in decline_texts())
    for total, k, texts in fill_calls():
        assert sum(len(x) for x in texts[:k]) == total
    groups = group_calls()
    assert sorted({len(g) for g in groups}) == [31, 32, 33, 63, 64, 65]


# ---------------------------------------------------------------- the oracle on synthetic vocabularies (checkable by hand)
@pytest.mark.parametrize("depth", [1, 3, 9])
def test_binary_chain_closed_form(depth):
    bpe = O.Bpe(chain_vocab_binary(depth))
    ns = list(range(0, 600))
    got = bpe.count([b"a" * n for n in ns])
    for n, g in zip(ns, got):
        assert int(g) == (n >> depth) + bin(n & ((1 << depth) - 1)).count("1"), (depth, n)


@pytest.mark.parametrize("k", [2, 5, 64, 512])
def test_linear_chain_closed_form(k):
    bpe = O.Bpe(chain_vocab_linear(k))
    ns = list(range(0, 600))
    got = bpe.count([b"a" * n for n in ns])
    for n, g in zip(ns, got):
        assert int(g) == -(-n // k), (k, n)
    # a space starts a new piece, so no merge crosses it: "aa" + " aa" = 1 + 2 tokens
    assert int(bpe.count([b"aa aa"])[0]) == 3


def test_duplicate_pair_keeps_first_rank():
    bpe = O.Bpe(duplicate_vocab())
    # abc: (a, b) at rank 0 merges before (b, c) at rank 1, then (300, c) -> 302: one token.  Were the repeat's rank 3 kept,
    # (b, c) would merge first and leave a + 301: two tokens
    assert [int(x) for x in bpe.count([b"abc", b"abbc", b"bb", b"ab"])] == [1, 2, 1, 1]


def test_collision_vocab_wraps_around():
    vocab, pairs = collision_vocab()
    slots = slots_for(len(vocab["merges"]))
    assert slots == 1024
    where = table_layout([tuple(m) for m in vocab["merges"]], slots)
    mask = slots - 1
    taken = sorted(where[(a << 16) | b] for a, b in pairs)
    # the nine pairs fill mask-2 .. mask and wrap to 0 .. 5 (unless other merges sit there first)
    assert mask in taken and 0 in taken
    assert any(where[(a << 16) | b] == mask and home(a, b, slots) != mask for a, b in pairs)   # a key probed into slot `mask`
    assert any(where[(a << 16) | b] < mask - 2 for a, b in pairs)                              # a key that wrapped around
    bpe = O.Bpe(vocab)
    assert all(int(c) == 1 for c in bpe.count([bytes([a, b]) for a, b in pairs]))


def test_largest_vocabulary_boundary():
    assert slots_for(4096) == 8192 and fits_shared_memory(4096)
    assert slots_for(4097) == 16384 and not fits_shared_memory(4097)
    v = largest_vocab(4096)
    keys = {(a << 16) | b for a, b, _ in v["merges"]}
    assert len(keys) == 4096 and max(m[2] for m in v["merges"]) == 256 + 4095


def test_high_ids_vocab_in_range():
    v = high_id_vocab()
    ids = v["byte_to_id"] + [x for m in v["merges"] for x in m]
    assert max(ids) == MAX_ID
    bpe = O.Bpe(v)
    # a b -> 65534, + c -> 65533; "ab ab" -> 65534 and " " + 65534 -> 65529: 2 tokens
    assert [int(x) for x in bpe.count([b"abc", b"ab ab", b"no", b"zz", b"ab" + b"ab"])] == [1, 2, 1, 1, 1]


# ---------------------------------------------------------------- request bodies for emb_scan_kernel
PAD = b"lorem ipsum dolor sit amet consectetur adipiscing elit sed do eiusmod tempor "


def pad(k: int, start: int = 0) -> bytes:
    reps = (start + k) // len(PAD) + 2
    return (PAD * reps)[start:start + k]


TAIL = b',"tail input","' + pad(60) + b'"]}'

# feature -> (builder of a body whose feature byte is at offset p or None when p is too small, expected outcome)
#   expected: "oracle" (status, model, inputs and tokens as the oracle says), or (DECLINED reason)
R_ESCAPE, R_CTRL_IN_STRING, R_TOO_LARGE, R_TOKENS, R_ARENA_FULL = 4, 3, 1, 5, 18
HEAD = b'{"model":"m","input":["'   # 23 bytes


def _tail_input(p):
    return b'"' + pad(40, p % 7) + b'"]}'


def feature_body(feature: str, p: int):
    H = len(HEAD)
    if feature == "open_quote":
        k = p - H - 2
        return None if k < 0 else HEAD + pad(k) + b'",' + b'"' + pad(50) + b'"]}'
    if feature == "close_quote":
        k = p - H
        return None if k < 0 else HEAD + pad(k) + b'"' + TAIL
    if feature == "comma":
        k = p - H - 1
        return None if k < 0 else HEAD + pad(k) + b'",' + _tail_input(p)
    if feature == "lbracket":      # the padding goes into "user": a model span is limited to 65535 bytes
        k = p - 19
        return None if k < 0 else b'{"user":"' + pad(k) + b'","input":[' + b'"' + pad(30) + b'"]}'
    if feature == "rbracket":
        k = p - H - 1
        return None if k < 0 else HEAD + pad(k) + b'"],"user":"' + pad(40) + b'"}'
    if feature == "colon":
        k = p - 18
        return None if k < 0 else b'{"user":"' + pad(k) + b'","input":["' + pad(30) + b'"]}'
    if feature in ("dimensions", "null", "true"):
        value, key = {"dimensions": (b"153600000", b"dimensions"), "null": (b"null", b"dimensions"), "true": (b"true", b"encoding_format")}[feature]
        mid = b'"],"' + key + b'":'
        k = p - H - len(mid)
        return None if k < 0 else HEAD + pad(k) + mid + value + b',"user":"' + pad(40) + b'"}'
    if feature == "whitespace":
        k = p - H - 1
        return None if k < 0 else HEAD + pad(k) + b'"' + b" \n\t\r  \n   " + b"," + b"\r\n  " + b'"' + pad(40) + b'"  ]  }  '
    if feature == "utf8":
        k = p - H
        return None if k < 0 else HEAD + pad(k) + "é日🙂".encode() + b" " + "日本語".encode() + b'"' + TAIL
    if feature == "backslash":
        k = p - H
        return None if k < 0 else HEAD + pad(k) + b"\\n" + b'"' + TAIL
    if feature == "ctrl_in_string":
        k = p - H
        return None if k < 0 else HEAD + pad(k) + b"\x01" + b'"' + TAIL
    if feature == "ctrl_outside":
        k = p - H - 1
        return None if k < 0 else HEAD + pad(k) + b'"' + b"\x01" + TAIL
    raise KeyError(feature)


def feature_offset(feature: str, body: bytes) -> int:
    """Where feature_body put the feature byte (recomputed from the body, to check the builder)."""
    if feature == "open_quote":
        return body.index(b'",', len(HEAD)) + 2
    if feature == "close_quote":
        return body.index(b'"', len(HEAD))
    if feature == "comma":
        return body.index(b'",', len(HEAD)) + 1
    if feature == "lbracket":
        return body.index(b"[")
    if feature == "rbracket":
        return body.index(b"]")
    if feature == "colon":
        return body.index(b'"input":') + 7
    if feature in ("dimensions", "null", "true"):
        return body.index(b'":', body.index(b"]")) + 2
    if feature == "whitespace":
        return body.index(b'"', len(HEAD)) + 1
    if feature == "utf8":
        return body.index("é".encode())
    if feature == "backslash":
        return body.index(b"\\")
    if feature in ("ctrl_in_string", "ctrl_outside"):
        return body.index(b"\x01")
    raise KeyError(feature)


FEATURES = ("open_quote", "close_quote", "comma", "lbracket", "rbracket", "colon", "dimensions", "null", "true", "whitespace", "utf8",
            "backslash", "ctrl_in_string", "ctrl_outside")
DECLINE_FEATURES = {"backslash": R_ESCAPE, "ctrl_in_string": R_CTRL_IN_STRING}
# thread, warp and tile boundaries on the 1st, 2nd and 8th tile
CENTERS = (THREAD_SPAN, WARP_SPAN, TILE, TILE + THREAD_SPAN, TILE + WARP_SPAN, 2 * TILE, 7 * TILE, 7 * TILE + THREAD_SPAN, 7 * TILE + WARP_SPAN, 8 * TILE)


def feature_positions():
    return sorted({c + d for c in CENTERS for d in range(-40, 41) if c + d >= 0})


def body_of_length(n: int, seed: int = 0) -> bytes:
    """{"input":["<pad>"]} of exactly n bytes (n >= 14)."""
    return b'{"input":["' + pad(n - 14, seed % 61) + b'"]}'


def tokens_body(n_tokens: int, n_bytes: int) -> bytes:
    """A valid request with exactly n_tokens scan tokens and exactly n_bytes bytes: k empty-ish inputs plus optional members that
    set the count modulo 3, the rest of the bytes as text inside the first input."""
    # {"input":[k strings]} is 3k + 6 tokens; "dimensions":1, adds 5 and "encoding_format":null, another 5
    extra, extra_tok = [(b"", 0), (b'"dimensions":1,"encoding_format":null,', 10), (b'"dimensions":1,', 5)][n_tokens % 3]
    k = (n_tokens - 6 - extra_tok) // 3
    assert k >= 1 and 3 * k + 6 + extra_tok == n_tokens
    fill = n_bytes - (1 + len(extra) + len(b'"input":[') + 3 * k - 1 + 2)
    assert fill >= 0, (n_tokens, n_bytes)
    return b"{" + extra + b'"input":[' + b",".join([b'"' + pad(fill) + b'"'] + [b'""'] * (k - 1)) + b"]}"


def scan_tokens(body: bytes) -> int:
    """emb_scan_kernel's token count for a body without backslashes: structural bytes outside strings, both quotes of every string,
    the first byte of every run of other non-whitespace bytes outside strings."""
    n, in_str, prev = 0, False, False
    for c in body:
        if c == 0x22:
            n += 1; in_str = not in_str; prev = False
        elif in_str:
            prev = False
        elif c in b"{}[]:,":
            n += 1; prev = False
        elif c in b" \t\n\r":
            prev = False
        else:
            n += not prev; prev = True
    return n


def request_inputs(body: bytes):
    """The input texts of an accepted request, as raw bytes (the accepted shape has no escapes)."""
    inp = json.loads(body).get("input")
    if inp is None:
        return []
    return [inp.encode()] if isinstance(inp, str) else [s.encode() for s in inp]


def test_feature_bodies_place_the_feature():
    for f in FEATURES:
        n = 0
        for p in feature_positions():
            b = feature_body(f, p)
            if b is None:
                continue
            assert feature_offset(f, b) == p, (f, p)
            n += 1
        assert n > 600, f


@pytest.mark.parametrize("f", FEATURES)
def test_feature_bodies_oracle_verdict(f):
    """The oracle's verdict on every feature body: OK or 400 as designed, and never a decline feature without its byte."""
    want = {"true": O.MALFORMED_400, "ctrl_outside": O.MALFORMED_400}.get(f, O.OK)
    for p in feature_positions()[::7]:
        b = feature_body(f, p)
        if b is None or f in DECLINE_FEATURES:
            continue
        t = O.embeddings_translate("openai", b)
        assert t.status == want, (f, p, t.err)


def test_length_bodies_and_token_bodies():
    for n in (14, 15, 100, 8191, 8192, 8193, 3 * 8192):
        assert len(body_of_length(n)) == n and json.loads(body_of_length(n))
    for t, n in ((306, 484), (307, 484), (308, 600), (3000, 6000), (3001, 6000), (3002, 6000)):
        b = tokens_body(t, n)
        assert len(b) == n and scan_tokens(b) == t, (t, n, len(b), scan_tokens(b))
        assert O.embeddings_translate("openai", b).status == O.OK
    assert scan_tokens(b'{"model":"m","input":["a b",""],"dimensions": 12 }') == 23   # { "model" : "m" , "input" : [ "a b" , "" ] , "dimensions" : 12 }
