// Per-document stage bodies of the chat translate pass, shared by the persistent throughput kernels (chat_kernel.cu) and the
// fused small-batch kernel (chat_walk_impl.cuh): index_doc (stages 2 + 2.5), emit_prefix / emit_doc (stage 5).  sm_90a only.
#pragma once
#include "chat_internal.cuh"
#include "classify.cuh"

namespace aigw {

// 16 bytes starting at an arbitrary shared-memory address (buffers carry ≥ 4 bytes of slack)
__device__ __forceinline__ uint4 lds16_unaligned(const uint8_t* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  const uint32_t sh = (a & 3u) * 8u;
  const uint32_t* w = (const uint32_t*)(p - (a & 3u));
  const uint32_t w0 = w[0], w1 = w[1], w2 = w[2], w3 = w[3], w4 = w[4];
  uint4 r;
  r.x = __funnelshift_r(w0, w1, sh); r.y = __funnelshift_r(w1, w2, sh); r.z = __funnelshift_r(w2, w3, sh); r.w = __funnelshift_r(w3, w4, sh);
  return r;
}

__device__ __forceinline__ aigw_doc_result blank_result(uint32_t len) {
  aigw_doc_result res;
  res.out_off = 0; res.body_len = 0; res.path_len = 0; res.status = AIGW_DECLINED; res.reason = AIGW_R_NONE;
  res.model_off = 0; res.model_len = 0; res.body_kind = AIGW_BODY_UNCHANGED; res.flags = 0; res.in_len = len; res._pad = 0;
  return res;
}
__device__ __forceinline__ uint32_t bin_of(uint32_t w) { const uint32_t n = w & 0x3fffffffu; return (w & 0x80000000u) ? 0u : (n < (uint32_t)kBins ? n : (uint32_t)kBins - 1u); }

// per-byte equality against a 7-bit constant as a most-significant-bit mask (0x80 per matching byte); z = w & 0x7f7f7f7f
__device__ __forceinline__ uint32_t eq_msb(uint32_t w, uint32_t z, uint32_t c4) { return ~(((z ^ c4) + 0x7f7f7f7fu) | w) & 0x80808080u; }
// bytes below 0x20
__device__ __forceinline__ uint32_t ctl_msb(uint32_t w, uint32_t z) { return ~((z + 0x60606060u) | w) & 0x80808080u; }
// msb mask → 4-bit mask (byte k → bit k): the four products land on bits 28..31 without carries
__device__ __forceinline__ uint32_t nib_from_msb(uint32_t t) { return (t * 0x00204081u) >> 28; }

// A round's sparse work (bytes outside strings, token compaction) is done cooperatively when few lanes own any of it:
// the owning lane's mask is broadcast and lane i handles its bit i, so a 28-byte cluster of punctuation between two
// messages costs one pass of ~12 instructions instead of a 28-trip single-lane loop.

// ---- stages 2 + 2.5 of one document, by one warp: structural index of the body staged at s_in[0, len) into token words
// s_tw[0, ntok) (position | byte | id / run length | escape flags).  Returns ntok (| bit 30: whitespace outside strings), or
// 0x80000000 | aigw_reason.
// s_bs: kTok halfwords (running backslash counts, later the lookup list); s_nc: one word per 1 KB round.
template <int MAXD>
__device__ __forceinline__ uint32_t index_doc(const uint8_t* s_in, uint32_t len, int lane, uint32_t* s_tw, uint16_t* s_bs, uint32_t* s_nc, const IdTables* s_ids) {
  using C = Cls<MAXD>;
  const uint32_t lt = (1u << lane) - 1u;
  const uint32_t rounds = (len + 1023u) >> 10;
  uint32_t carry_esc = 0, carry_str = 0, carry_sc = 0;
  uint32_t ntok = 0, bs_run = 0;
  uint32_t flags = 0;  // bit0 ctrl in string, bit1 bad escape, bit2 token overflow
  uint32_t any_nc = 0; // some round holds a valid escape the encoder re-spells (warp-uniform)
  uint32_t ws_any = 0; // whitespace outside strings (per lane; reduced at the end)
  for (uint32_t r = 0; r < rounds; r++) {
    const uint32_t rbase = r << 10;
    const uint32_t base = rbase + (lane << 5);
    // bytes at or beyond len (stale shared memory) are masked out of every class
    const uint32_t valid = base + 32u <= len ? 0xffffffffu : (base >= len ? 0u : ((1u << (len - base)) - 1u));
    const uint4 a = *(const uint4*)(s_in + base), b = *(const uint4*)(s_in + base + 16);
    const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    // every class mask of the lane's 32 bytes at once (classify.cuh: 8 bit planes, then LOP3s)
    const ByteClasses bc = classify32(w);
    const uint32_t mq = bc.quote & valid, mb = bc.bslash & valid, mctl = bc.ctl & valid;
    // escaped characters: odd-length backslash runs, carry across lanes
    uint32_t esc = 0, bs_lane = 0;
    const uint32_t any_bs = __ballot_sync(FULL, mb != 0);
    if (any_bs | carry_esc) {
      const uint32_t tail = __clz(~mb);  // backslash run length at the top of this lane's 32 bytes
      const uint32_t odd = __ballot_sync(FULL, tail < 32u && (tail & 1u));
      const uint32_t full = __ballot_sync(FULL, tail == 32u);
      uint32_t cin;
      {
        const uint32_t below = ~full & lt;
        if (below == 0) cin = carry_esc; else cin = (odd >> (31 - __clz(below))) & 1u;
      }
      {
        const uint32_t below = ~full;
        carry_esc = below == 0 ? carry_esc : (odd >> (31 - __clz(below))) & 1u;
      }
      const uint32_t bs = mb & ~cin;  // a leading backslash that is itself escaped starts no run
      const uint32_t follows = (bs << 1) | cin;
      const uint32_t even = 0x55555555u;
      const uint32_t odd_starts = bs & ~even & ~follows;
      const uint32_t seq_even = odd_starts + bs;  // carry-out handled through `tail`
      const uint32_t invert = seq_even << 1;
      esc = (even ^ invert) & follows;
      // running backslash count in front of this lane (tokens remember it: a string has an escape iff the count moves)
      const uint32_t pc = __popc(mb);
      uint32_t incl = pc;
#pragma unroll
      for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, sft); if (lane >= sft) incl += v; }
      bs_lane = bs_run + incl - pc;
      bs_run += __shfl_sync(FULL, incl, 31);
    } else bs_lane = bs_run;
    esc &= valid;
    const uint32_t uq = mq & ~esc;
    uint32_t ps = uq;
    ps ^= ps << 1; ps ^= ps << 2; ps ^= ps << 4; ps ^= ps << 8; ps ^= ps << 16;
    const uint32_t par = __ballot_sync(FULL, __popc(uq) & 1);
    const uint32_t sin = (__popc(par & lt) & 1u) ^ carry_str;
    if (sin) ps = ~ps;
    carry_str ^= __popc(par) & 1u;
    ps &= valid;
    // ps: bit set from an opening quote up to the byte before its closing quote
    if (mctl & ps) flags |= 1u;
    {  // escaped characters: \" \\ \n \r \t are what the encoder writes back; \/ \b \f \uXXXX are valid but re-spelled (marked per
       // 32-byte block, re-escaped by the walk when the string is echoed); anything else is not JSON
      uint32_t e = esc & ps; bool nc = false;
      while (e) {
        const int j = __ffs(e) - 1; e &= e - 1; const uint32_t c = s_in[base + j];
        if (!(c == '"' || c == '\\' || c == 'n' || c == 'r' || c == 't')) { if (c == '/' || c == 'b' || c == 'f' || c == 'u') nc = true; else flags |= 2u; }
      }
      const uint32_t ncm = __ballot_sync(FULL, nc);
      if (lane == 0) s_nc[r] = ncm;
      any_nc |= ncm;
    }
    // bytes outside strings: structural characters are tokens, everything that is neither structural nor whitespace is a
    // scalar character (a control character other than \t \n \r lands there and fails the scalar grammar in the walk)
    const uint32_t outside = ~ps & ~uq & valid;
    ws_any |= outside & bc.ws;
    uint32_t mtok = uq | (bc.op & outside);
    const uint32_t msc = outside & ~bc.op & ~bc.ws;
    {
      uint32_t prev = __shfl_up_sync(FULL, msc >> 31, 1);
      if (lane == 0) prev = carry_sc;
      carry_sc = __shfl_sync(FULL, msc >> 31, 31);
      mtok |= msc & ~((msc << 1) | prev);
    }
    // compact token words: position | byte | (scalars) length of the run inside this 32-byte block
    const uint32_t cnt = __popc(mtok);
    uint32_t incl = cnt;
#pragma unroll
    for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, sft); if (lane >= sft) incl += v; }
    const uint32_t total = __shfl_sync(FULL, incl, 31);
    const uint32_t wpos0 = ntok + incl - cnt;
    if (ntok + total > (uint32_t)C::kTok) flags |= 4u;
    else {
      const uint32_t tl = __ballot_sync(FULL, mtok != 0);
      if (17u * (uint32_t)__popc(tl) <= 13u * __reduce_max_sync(FULL, cnt)) {   // ≈ instructions per owning lane vs per trip of the per-lane loop
        uint32_t m = tl;
        while (m) {
          const int L = __ffs(m) - 1; m &= m - 1;
          const uint32_t mk = __shfl_sync(FULL, mtok, L), wq = __shfl_sync(FULL, wpos0, L), sc = __shfl_sync(FULL, msc, L);
          const uint32_t mbL = __shfl_sync(FULL, mb, L), bsL = __shfl_sync(FULL, bs_lane, L);
          if ((mk >> lane) & 1u) {
            const uint32_t pos = rbase + (L << 5) + lane;
            uint32_t tword = pos | ((uint32_t)s_in[pos] << 16);
            if ((sc >> lane) & 1u) { const uint32_t run = __ffs(~(sc >> lane)) - 1u; if (lane + run < 32u) tword |= run << 24; }  // a run that reaches the block end is measured by the walker
            const uint32_t slot = wq + __popc(mk & lt);
            s_tw[slot] = tword;
            s_bs[slot] = (uint16_t)(bsL + __popc(mbL & lt));
          }
        }
      } else {
        uint32_t m = mtok, wpos = wpos0;
        while (m) {
          const int j = __ffs(m) - 1; m &= m - 1;
          uint32_t tword = (base + j) | ((uint32_t)s_in[base + j] << 16);
          if ((msc >> j) & 1u) { const uint32_t run = __ffs(~(msc >> j)) - 1u; if (j + run < 32u) tword |= run << 24; }
          s_tw[wpos] = tword;
          s_bs[wpos] = (uint16_t)(bs_lane + __popc(mb & ((1u << j) - 1u)));
          wpos++;
        }
      }
    }
    ntok += total;
  }
  flags = __reduce_or_sync(FULL, flags);
  __syncwarp();
  int reason = 0;
  if (flags & 4u) reason = AIGW_R_TOKENS;
  else if (flags & 1u) reason = AIGW_R_CTRL_IN_STRING;
  else if (flags & 2u) reason = AIGW_R_ESCAPE;
  else if (carry_str) reason = AIGW_R_E400_SYNTAX;
  if (reason) return 0x80000000u | (uint32_t)reason;
  // ---- stage 2.5: strings get their escape flag and (short, unescaped ones) a key / value id.  Quote tokens alternate
  // open/close, so opening quotes are the quote tokens of even rank.  Pass 1 (one token per lane) collects the strings worth
  // a lookup into a dense list, pass 2 runs the hash lookup with every lane busy.
  uint32_t nlk = 0;
  {
    uint16_t* s_lk = s_bs;   // list entry k ≤ i/2 never overtakes the counts still to be read (same-iteration reads are fenced)
    uint32_t qbase = 0;
    for (uint32_t b0 = 0; b0 < ntok; b0 += 32) {
      const uint32_t i = b0 + lane;
      const uint32_t w = i < ntok ? s_tw[i] : 0u;
      const bool isq = i < ntok && ((w >> 16) & 0xffu) == '"';
      const uint32_t qm = __ballot_sync(FULL, isq);
      bool want = false;
      if (isq && ((qbase + __popc(qm & lt)) & 1u) == 0 && i + 1 < ntok) {
        const uint32_t o = (w & 0xffffu) + 1u, n = (s_tw[i + 1] & 0xffffu) - o;
        const bool esc = s_bs[i + 1] != s_bs[i];
        if (esc) {
          uint32_t ncf = 0, id = 0;
          if (any_nc) {   // only documents that hold a re-spelled escape pay for the per-string questions
            // bit 31: some block the string touches holds a re-spelled escape (conservative: the walk re-checks byte by byte)
            const uint32_t b0k = o >> 5, b1k = (o + n) >> 5;
            for (uint32_t wk = b0k >> 5; wk <= (b1k >> 5); wk++) {
              uint32_t m = s_nc[wk];
              if (wk == (b0k >> 5)) m &= ~0u << (b0k & 31u);
              if (wk == (b1k >> 5)) m &= (b1k & 31u) == 31u ? ~0u : ((2u << (b1k & 31u)) - 1u);
              ncf |= m;
            }
            // ids are looked up on the decoded bytes, so an escaped spelling of a key or of an enumerated value keeps its meaning
            // (a string whose escapes are all canonical cannot equal a table entry: none contains such a character)
            if (ncf && n <= 6u * (uint32_t)kMaxIdLen) { const bool is_key = i + 2 < ntok && ((s_tw[i + 2] >> 16) & 0xffu) == ':'; id = lookup_id_escaped(s_ids, s_in + o, n, is_key); }
          }
          s_tw[i] = w | (1u << 30) | (ncf ? (1u << 31) : 0u) | (id << 24);
        }
        want = !esc && n >= 1u && n <= (uint32_t)kMaxIdLen;
      }
      __syncwarp();
      const uint32_t wm = __ballot_sync(FULL, want);
      if (want) s_lk[nlk + __popc(wm & lt)] = (uint16_t)i;
      nlk += __popc(wm);
      qbase += __popc(qm);
    }
    __syncwarp();
    for (uint32_t k = lane; k < nlk; k += 32) {
      const uint32_t i = s_lk[k];
      const uint32_t w = s_tw[i];
      const uint32_t o = (w & 0xffffu) + 1u, n = (s_tw[i + 1] & 0xffffu) - o;
      const bool is_key = i + 2 < ntok && ((s_tw[i + 2] >> 16) & 0xffu) == ':';
      s_tw[i] = w | (lookup_id(s_ids, s_in + o, n, is_key) << 24);
    }
    __syncwarp();
  }
  // bit 30: some byte outside strings is whitespace (the /v1/messages planner needs to know whether the body is compact)
  return ntok | (__any_sync(FULL, ws_any != 0) ? 0x40000000u : 0u);
}

static constexpr int kEmitTile = 256;   // chunks per tile of the op-start table
template <int MAXD>
struct EmitSmem {
  using C = Cls<MAXD>;
  static constexpr int kPreB = (C::kOps + 4) * 4, kOpsB = C::kOps * 4, kScrB = (C::kScr + 15) & ~15, kFirstB = kEmitTile * 2, kBlB = (C::kOps + 4) * 4;
  static constexpr int kWarpBytes = C::kIn + kPreB + kOpsB + kScrB + kFirstB + kBlB;
};


// ---- stage 5 helpers.  emit_prefix: ops (+ exclusive prefix of their lengths) into shared memory; returns the scratch bytes
// the ops reference.  gops may be global (the walk kernel's plan) or shared (fused small-batch kernel).
template <int MAXD>
__device__ __forceinline__ uint32_t emit_prefix(const uint32_t* gops, uint32_t op_first, uint32_t nops, uint32_t olen, uint32_t* s_ops, uint32_t* s_pre, int lane) {
  uint32_t run = 0, scr_hi = 0;
  for (uint32_t b0 = 0; b0 < nops; b0 += 32) {
    const uint32_t k = b0 + lane;
    const uint32_t op = k < nops ? (b0 == 0 ? op_first : gops[k]) : 0u;
    const uint32_t l = (op >> 16) & 0x3fffu;
    if ((op >> 30) == 2u) scr_hi = max(scr_hi, (op & 0xffffu) + l);
    uint32_t incl = l;
#pragma unroll
    for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, sft); if (lane >= sft) incl += v; }
    if (k < nops) { s_ops[k] = op; s_pre[k] = run + incl - l; }
    run += __shfl_sync(FULL, incl, 31);
  }
  if (lane == 0) s_pre[nops] = olen;
  return __reduce_max_sync(FULL, scr_hi);
}

// emit_doc: the output record as 16-byte chunks, one chunk per lane (see the emit kernel's header comment)
template <int MAXD>
__device__ __forceinline__ void emit_doc(const uint8_t* s_in, const uint8_t* s_lits, const uint8_t* s_scr, const uint32_t* s_pre, const uint32_t* s_ops, uint16_t* s_first, uint32_t* s_bl,
                                         uint32_t nops, uint32_t nchunks, uint4* o4, int lane) {
  const uint32_t lt = (1u << lane) - 1u;
  uint32_t carry = 0, nb = 0;
  for (uint32_t t0 = 0; t0 < nchunks; t0 += kEmitTile) {
    const uint32_t tn = min((uint32_t)kEmitTile, nchunks - t0);
    for (uint32_t i = lane; i < (tn + 1u) >> 1; i += 32) ((uint32_t*)s_first)[i] = 0u;
    __syncwarp();
    // op k is the last op that starts in (16(c-1), 16c] ⇒ it owns the table entry of chunk c
    for (uint32_t k = lane; k < nops; k += 32) {
      const uint32_t c = (s_pre[k] + 15u) >> 4, cn = (s_pre[k + 1] + 15u) >> 4;
      if (c != cn && c - t0 < tn) s_first[c - t0] = (uint16_t)k;
    }
    __syncwarp();
    for (uint32_t i0 = 0; i0 < tn; i0 += 32) {
      const uint32_t i = i0 + lane;
      const bool valid = i < tn;
      uint32_t k = valid ? (uint32_t)s_first[i] : 0u;
#pragma unroll
      for (int sft = 1; sft < 32; sft <<= 1) k = max(k, __shfl_up_sync(FULL, k, sft));
      k = max(k, carry);
      carry = __shfl_sync(FULL, k, 31);
      const uint32_t c = t0 + i, pos = c << 4;
      const uint32_t p0 = s_pre[k], p1 = s_pre[k + 1];
      const bool interior = valid && p1 >= pos + 16u;
      if (interior) {
        const uint32_t op = s_ops[k];
        const uint32_t kind = op >> 30, off = op & 0xffffu;
        const uint8_t* sp = (kind == 0 ? s_in : kind == 1 ? s_lits : s_scr) + off + (pos - p0);
        o4[c] = lds16_unaligned(sp);
      }
      const bool edge = valid && !interior;
      const uint32_t bm = __ballot_sync(FULL, edge);
      if (edge) s_bl[nb + __popc(bm & lt)] = c | (k << 16);
      nb += __popc(bm);
    }
    __syncwarp();
  }
  // chunks that straddle op boundaries: OR together one shifted, masked 16-byte read per overlapping op
  for (uint32_t bi = lane; bi < nb; bi += 32) {
    const uint32_t ent = s_bl[bi];
    const uint32_t c = ent & 0xffffu, pos = c << 4;
    uint32_t k = ent >> 16;
    uint32_t op = s_ops[k];
    uint32_t kind = op >> 30, l = (op >> 16) & 0x3fffu, off = op & 0xffffu;
    uint32_t within = pos - s_pre[k];
    const uint8_t* sp = (kind == 0 ? s_in : kind == 1 ? s_lits : s_scr) + off;
    uint4 v = make_uint4(0, 0, 0, 0);
    uint32_t filled = 0;
    for (;;) {
      if (within >= l) {
        if (++k >= nops) break;
        op = s_ops[k]; kind = op >> 30; l = (op >> 16) & 0x3fffu; off = op & 0xffffu; within = 0;
        sp = (kind == 0 ? s_in : kind == 1 ? s_lits : s_scr) + off;
        continue;
      }
      const uint32_t take = min(l - within, 16u - filled);
      uint4 x = lds16_unaligned(sp + within);
      {  // keep the first `take` bytes
        const uint32_t t0 = take, t1 = take > 4u ? take - 4u : 0u, t2 = take > 8u ? take - 8u : 0u, t3 = take > 12u ? take - 12u : 0u;
        x.x &= t0 >= 4u ? 0xffffffffu : ((1u << (8u * t0)) - 1u);
        x.y &= t1 >= 4u ? 0xffffffffu : ((1u << (8u * t1)) - 1u);
        x.z &= t2 >= 4u ? 0xffffffffu : ((1u << (8u * t2)) - 1u);
        x.w &= t3 >= 4u ? 0xffffffffu : ((1u << (8u * t3)) - 1u);
      }
      {  // shift left by `filled` bytes (128-bit) and merge
        const uint32_t bsh = (filled & 3u) * 8u, wsh = filled >> 2;
        const uint32_t r0 = x.x << bsh, r1 = __funnelshift_l(x.x, x.y, bsh), r2 = __funnelshift_l(x.y, x.z, bsh), r3 = __funnelshift_l(x.z, x.w, bsh);
        if (wsh == 0) { v.x |= r0; v.y |= r1; v.z |= r2; v.w |= r3; }
        else if (wsh == 1) { v.y |= r0; v.z |= r1; v.w |= r2; }
        else if (wsh == 2) { v.z |= r0; v.w |= r1; }
        else v.w |= r0;
      }
      filled += take; within += take;
      if (filled >= 16u) break;
    }
    o4[c] = v;
  }
}

}  // namespace aigw
