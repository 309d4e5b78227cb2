// See mutate_kernel.cuh.  sm_90a only.
#include "device_once.cuh"
#include "mutate_kernel.cuh"

namespace aigw {
namespace {

constexpr uint32_t FULLM = 0xffffffffu;
constexpr int kMem = 128;      // top-level members handled per body
constexpr int kPieces = 96;    // copy pieces per body
constexpr uint32_t kText = 0x80000000u;

__device__ __forceinline__ uint32_t nib_from_ff(uint32_t m) { return ((m & 0x08040201u) * 0x01010101u) >> 24; }
__device__ __forceinline__ bool ws(uint32_t c) { return c == ' ' || c == '\n' || c == '\r' || c == '\t'; }
__device__ __forceinline__ uint32_t bits_range(uint32_t lo, uint32_t hi) {  // bits [lo, hi), 0 ≤ lo ≤ hi ≤ 32
  const uint32_t a = hi >= 32u ? 0xffffffffu : ((1u << hi) - 1u);
  const uint32_t b = lo >= 32u ? 0xffffffffu : ((1u << lo) - 1u);
  return a & ~b;
}

// whether the copy pieces spell the staged input; called by the whole warp, out of line so the copy path's code stays as it was
__device__ __noinline__ bool pieces_equal_input(const uint8_t* s_text, const uint8_t* s_in, const uint32_t* s_psrc, const uint32_t* s_plen,
                                                uint32_t np, int lane) {
  uint32_t diff = 0, o = 0;
  for (uint32_t p = 0; p < np; p++) {
    const uint32_t src = s_psrc[p], l = s_plen[p];
    const uint8_t* sp = (src & kText) ? s_text + (src & ~kText) : s_in + src;
    for (uint32_t i = lane; i < l; i += 32) diff |= sp[i] != s_in[o + i];
    o += l;
  }
  return !__any_sync(FULLM, diff);
}

template <int MAXD>
struct Lay {
  static constexpr int kIn = ((MAXD + 1023) / 1024) * 1024 + 16;
  static constexpr int kWarpBytes = kIn + (kMem + 4) * 4 + kMem * 16 + kPieces * 8;
};

template <int MAXD, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) body_mutate_kernel(const __grid_constant__ MutateParams P) {
  using L = Lay<MAXD>;
  extern __shared__ __align__(16) uint8_t smem[];
  uint8_t* s_text = smem;                       // key names, `"key":value` members, replacement values, one ','
  uint8_t* s_cls = smem + kMutTextCap;          // 1 open, 2 close, 3 comma, 4 whitespace
  for (uint32_t i = threadIdx.x; i < kMutTextCap / 4; i += blockDim.x) ((uint32_t*)s_text)[i] = ((const uint32_t*)P.text)[i];
  for (uint32_t c = threadIdx.x; c < 256; c += blockDim.x) s_cls[c] = (c == '{' || c == '[') ? 1 : (c == '}' || c == ']') ? 2 : c == ',' ? 3 : ws(c) ? 4 : 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* wb = smem + kMutTextCap + 256 + (size_t)warp * L::kWarpBytes;
  uint8_t* s_in = wb;
  uint32_t* s_sep = (uint32_t*)(wb + L::kIn);
  uint4* s_mem = (uint4*)(s_sep + kMem + 4);
  uint32_t* s_psrc = (uint32_t*)(s_mem + kMem);
  uint32_t* s_plen = s_psrc + kPieces;
  const uint32_t comma_off = kMutTextCap - 4;   // the host puts ',' there

  for (;;) {
    uint32_t doc = 0;
    if (lane == 0) doc = atomicAdd(P.next, 1u);
    doc = __shfl_sync(FULLM, doc, 0);
    if (doc >= P.n) break;
    const uint32_t len = P.lens[doc];
    aigw_mut_result res; res.out_off = 0; res.out_len = 0; res.status = AIGW_DECLINED; res.reason = AIGW_R_NONE; res.flags = 0;
    if (len == 0 || len > (uint32_t)MAXD) { res.reason = len ? AIGW_R_TOO_LARGE : AIGW_R_SYNTAX; if (lane == 0) P.results[doc] = res; continue; }
    // ---- stage the body, pad the last round with spaces
    const uint32_t rounds = (len + 1023u) >> 10;
    {
      const uint8_t* g = P.bodies + P.offsets[doc];
      const uint32_t mis = (uint32_t)((uintptr_t)g & 15u);
      if (mis == 0) {
        const uint4* g4 = (const uint4*)g; uint4* s4 = (uint4*)s_in;
        for (uint32_t i = lane; i < ((len + 15u) >> 4); i += 32) s4[i] = __ldg(g4 + i);
      } else {
        for (uint32_t i = lane; i < len; i += 32) s_in[i] = g[i];
      }
      __syncwarp();
      for (uint32_t i = len + lane; i < (rounds << 10); i += 32) s_in[i] = ' ';
      __syncwarp();
    }
    // ---- stage A: member separators (root braces and depth-1 commas)
    uint32_t carry_esc = 0, carry_str = 0;
    int depth = 0;
    uint32_t nsep = 0, ws_top = 0, overflow = 0;
    for (uint32_t r = 0; r < rounds; r++) {
      const uint32_t base = (r << 10) + ((uint32_t)lane << 5);
      const uint4 a = *(const uint4*)(s_in + base), b = *(const uint4*)(s_in + base + 16);
      const uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      uint32_t mq = 0, mb = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) {
        mq |= nib_from_ff(__vcmpeq4(w[j], 0x22222222u)) << (4 * j);
        mb |= nib_from_ff(__vcmpeq4(w[j], 0x5c5c5c5cu)) << (4 * j);
      }
      uint32_t esc = 0;
      const uint32_t any_bs = __ballot_sync(FULLM, mb != 0);
      if (any_bs | carry_esc) {   // escaped characters: odd-length backslash runs, carried across lanes and rounds
        const uint32_t tail = __clz(~mb);
        const uint32_t odd = __ballot_sync(FULLM, tail < 32u && (tail & 1u));
        const uint32_t full = __ballot_sync(FULLM, tail == 32u);
        uint32_t cin;
        { const uint32_t below = ~full & ((1u << lane) - 1u); cin = below == 0 ? carry_esc : (odd >> (31 - __clz(below))) & 1u; }
        { const uint32_t below = ~full; carry_esc = below == 0 ? carry_esc : (odd >> (31 - __clz(below))) & 1u; }
        const uint32_t bs = mb & ~cin;
        const uint32_t follows = (bs << 1) | cin;
        const uint32_t even = 0x55555555u;
        const uint32_t odd_starts = bs & ~even & ~follows;
        const uint32_t seq_even = odd_starts + bs;
        esc = (even ^ (seq_even << 1)) & follows;
      }
      const uint32_t uq = mq & ~esc;
      uint32_t ps = uq;
      ps ^= ps << 1; ps ^= ps << 2; ps ^= ps << 4; ps ^= ps << 8; ps ^= ps << 16;
      const uint32_t par = __ballot_sync(FULLM, __popc(uq) & 1);
      if ((__popc(par & ((1u << lane) - 1u)) & 1u) ^ carry_str) ps = ~ps;
      carry_str ^= __popc(par) & 1u;
      // structural bytes outside strings
      uint32_t mo = 0, mc = 0, mcm = 0, mws = 0;
      {
        uint32_t o = ~ps & ~uq;
        while (o) {
          const int j = __ffs(o) - 1; o &= o - 1;
          const uint32_t cl = s_cls[s_in[base + j]];
          if (cl == 4) mws |= 1u << j; else if (cl == 1) mo |= 1u << j; else if (cl == 2) mc |= 1u << j; else if (cl == 3) mcm |= 1u << j;
        }
      }
      int incl = __popc(mo) - __popc(mc);
      const int mine = incl;
#pragma unroll
      for (int sft = 1; sft < 32; sft <<= 1) { const int v = __shfl_up_sync(FULLM, incl, sft); if (lane >= sft) incl += v; }
      int d = depth + incl - mine;
      depth += __shfl_sync(FULLM, incl, 31);
      uint32_t sepm = 0, d1 = 0, prev = 0;
      {
        uint32_t ev = mo | mc | mcm;
        while (ev) {
          const uint32_t j = __ffs(ev) - 1; ev &= ev - 1;
          if (d == 1) d1 |= bits_range(prev, j);
          const uint32_t bit = 1u << j;
          if (mo & bit) { if (d == 0) sepm |= bit; d++; }
          else if (mc & bit) { d--; if (d == 0) sepm |= bit; }
          else if (d == 1) sepm |= bit;
          prev = j + 1;
        }
        if (d == 1) d1 |= bits_range(prev, 32);
      }
      if (mws & d1) ws_top = 1;
      uint32_t cnt = __popc(sepm), pre = cnt;
#pragma unroll
      for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t v = __shfl_up_sync(FULLM, pre, sft); if (lane >= sft) pre += v; }
      const uint32_t tot = __shfl_sync(FULLM, pre, 31);
      uint32_t wpos = nsep + pre - cnt;
      if (nsep + tot > (uint32_t)kMem + 1u) overflow = 1;
      else { uint32_t m = sepm; while (m) { const int j = __ffs(m) - 1; m &= m - 1; s_sep[wpos++] = base + j; } }
      nsep += tot;
    }
    ws_top = __any_sync(FULLM, ws_top);
    __syncwarp();
    int reason = 0;
    if (overflow) reason = AIGW_R_TOKENS;
    else if (carry_str || depth != 0 || nsep < 2) reason = AIGW_R_SYNTAX;
    else if (s_in[s_sep[0]] != '{' || s_in[s_sep[nsep - 1]] != '}') reason = AIGW_R_ROOT;
    if (!reason) {  // only whitespace outside the root object, only commas between the braces
      uint32_t bad = 0;
      for (uint32_t i = lane; i < s_sep[0]; i += 32) if (!ws(s_in[i])) bad = 1;
      for (uint32_t i = s_sep[nsep - 1] + 1 + lane; i < len; i += 32) if (!ws(s_in[i])) bad = 1;
      for (uint32_t i = 1 + lane; i + 1 < nsep; i += 32) if (s_in[s_sep[i]] != ',') bad = 1;
      if (__any_sync(FULLM, bad)) reason = AIGW_R_SYNTAX;
    }
    if (reason) { res.reason = (uint8_t)reason; if (lane == 0) P.results[doc] = res; continue; }
    // ---- stage B: one lane per member: "key" : value, key table match
    uint32_t nmem = nsep - 1;
    uint32_t found = 0, dup = 0, any_del = 0, bad_member = 0;
    for (uint32_t m0 = 0; m0 < nmem; m0 += 32) {
      const uint32_t i = m0 + lane;
      int match = -1; uint32_t act = 0;
      if (i < nmem) {
        const uint32_t s = s_sep[i] + 1, e = s_sep[i + 1];
        uint32_t p = s;
        while (p < e && ws(s_in[p])) p++;
        uint32_t vb = 0, ve = 0;
        if (p >= e) { if (!(nmem == 1)) bad_member = 1; else act = 3; }   // `{ }`: an empty object, not a member
        else if (s_in[p] != '"') bad_member = 1;
        else {
          const uint32_t ks = p + 1; uint32_t q = ks;
          while (q < e && s_in[q] != '"') { if (s_in[q] == '\\') bad_member = 2; q++; }
          const uint32_t kl = q - ks;
          p = q + 1;
          while (p < e && ws(s_in[p])) p++;
          if (p >= e || s_in[p] != ':') bad_member |= 1;
          p++;
          while (p < e && ws(s_in[p])) p++;
          vb = p; ve = e;
          while (ve > vb && ws(s_in[ve - 1])) ve--;
          if (vb >= ve) bad_member |= 1;
          for (uint32_t k = 0; k < P.n_keys; k++) {
            const MutateKey& K = P.keys[k];
            if (K.name_len != kl) continue;
            uint32_t t = 0; while (t < kl && s_in[ks + t] == s_text[K.name_off + t]) t++;
            if (t == kl) { match = (int)k; act = K.remove ? 1u : 2u; break; }
          }
        }
        s_mem[i] = make_uint4(s, vb, ve, act | ((uint32_t)(match & 0xff) << 8));
      }
      for (uint32_t k = 0; k < P.n_keys; k++) {
        const uint32_t bal = __ballot_sync(FULLM, match == (int)k);
        if (bal) { if ((found >> k) & 1u || __popc(bal) > 1) dup = 1; found |= 1u << k; }
      }
      if (__any_sync(FULLM, act == 1u)) any_del = 1;
    }
    bad_member = __reduce_or_sync(FULLM, bad_member);
    const bool empty_obj = nmem == 1 && (s_mem[0].w & 0xffu) == 3u;
    if (empty_obj) nmem = 0;
    if (bad_member) reason = (bad_member & 2u) ? AIGW_R_ESCAPE : AIGW_R_SYNTAX;
    else if (dup) reason = AIGW_R_DUP_KEY;
    else if (any_del && ws_top) reason = AIGW_R_UNSUPPORTED_FIELD;   // which comma sjson takes would show
    if (reason) { res.reason = (uint8_t)reason; if (lane == 0) P.results[doc] = res; continue; }
    __syncwarp();
    // ---- stage C: lane 0 folds the member actions into copy pieces
    uint32_t np = 0, total = 0, perr = 0, changed = 0;
    if (lane == 0) {
      auto put = [&](uint32_t src, uint32_t l) { if (!l) return; if (np >= (uint32_t)kPieces) { perr = 1; return; } s_psrc[np] = src; s_plen[np] = l; np++; total += l; };
      uint32_t app = 0;   // keys to append: set, and either absent or removed first
      for (uint32_t k = 0; k < P.n_keys; k++) if (P.keys[k].set && (!((found >> k) & 1u) || P.keys[k].remove)) app |= 1u << k;
      const uint32_t root_open = s_sep[0], root_close = s_sep[nsep - 1];
      long long cur = app ? (long long)root_open : 0;   // start of the open input run, -1 when none
      uint32_t alive = 0;
      for (uint32_t i = 0; i < nmem; i++) {
        const uint4 m = s_mem[i];
        const uint32_t act = m.w & 0xffu, k = (m.w >> 8) & 0xffu;
        if (act == 1u) {
          changed = 1;
          if (cur >= 0) { put((uint32_t)cur, s_sep[i] + (alive == 0 ? 1u : 0u) - (uint32_t)cur); cur = -1; }
        } else {
          if (cur < 0) { if (alive) put(kText | comma_off, 1); cur = m.x; }
          if (act == 2u) { changed = 1; put((uint32_t)cur, m.y - (uint32_t)cur); put(kText | P.keys[k].val_off, P.keys[k].val_len); cur = m.z; }
          alive++;
        }
      }
      if (!app) { if (cur < 0) cur = root_close; put((uint32_t)cur, len - (uint32_t)cur); }
      else {
        changed = 1;
        if (cur >= 0) put((uint32_t)cur, root_close - (uint32_t)cur);
        bool before = alive > 0;
        for (uint32_t k = 0; k < P.n_keys; k++) if ((app >> k) & 1u) { if (before) put(kText | comma_off, 1); put(kText | P.keys[k].memb_off, P.keys[k].memb_len); before = true; }
        put(root_close, 1);
      }
    }
    np = __shfl_sync(FULLM, np, 0); total = __shfl_sync(FULLM, total, 0); perr = __shfl_sync(FULLM, perr, 0); changed = __shfl_sync(FULLM, changed, 0);
    // flags bit0: the record is the input byte for byte.  Edits can rebuild it (a set to the value already there, a delete
    // whose re-append lands on the same bytes), so a record of the input's length is compared with the staged input below.
    const uint32_t same_rule = !changed ? 1u : total == len ? 2u : 0u;   // 1 identical, 2 compare, 0 different
    if (perr) { res.reason = AIGW_R_OPS; if (lane == 0) P.results[doc] = res; continue; }
    const uint32_t rec = (total + 15u) & ~15u;
    unsigned long long obase = 0;
    if (lane == 0) obase = atomicAdd(P.out_used, (unsigned long long)rec);
    obase = __shfl_sync(FULLM, obase, 0);
    if (obase + rec > P.out_capacity) { res.reason = AIGW_R_ARENA_FULL; if (lane == 0) P.results[doc] = res; continue; }
    __syncwarp();
    {
      uint8_t* dst = P.out + obase;
      uint32_t o = 0;
      for (uint32_t p = 0; p < np; p++) {
        const uint32_t src = s_psrc[p], l = s_plen[p];
        const uint8_t* sp = (src & kText) ? s_text + (src & ~kText) : s_in + src;
        // word copies when source and destination agree modulo 4 once the head is done, bytes otherwise
        uint8_t* dp = dst + o;
        if (l >= 64u && ((((uintptr_t)sp) ^ ((uintptr_t)dp)) & 3u) == 0) {
          uint32_t head = (uint32_t)((4u - ((uintptr_t)dp & 3u)) & 3u);
          if ((uint32_t)lane < head) dp[lane] = sp[lane];
          const uint32_t nw = (l - head) >> 2;
          const uint32_t* s32 = (const uint32_t*)(sp + head); uint32_t* d32 = (uint32_t*)(dp + head);
          for (uint32_t i = lane; i < nw; i += 32) d32[i] = s32[i];
          for (uint32_t i = head + (nw << 2) + lane; i < l; i += 32) dp[i] = sp[i];
        } else {
          for (uint32_t i = lane; i < l; i += 32) dp[i] = sp[i];
        }
        o += l;
      }
    }
    const bool same = same_rule == 1u || (same_rule == 2u && pieces_equal_input(s_text, s_in, s_psrc, s_plen, np, lane));
    res.out_off = obase + P.out_bias; res.out_len = total; res.status = AIGW_OK; res.flags = same ? 1 : 0;
    if (lane == 0) P.results[doc] = res;
    __syncwarp();
  }
}

template <int MAXD, int WARPS>
cudaError_t launch_cls(const MutateParams& P, int sm_count, cudaStream_t st) {
  static DeviceOnce once;
  const size_t smem = kMutTextCap + 256 + (size_t)WARPS * Lay<MAXD>::kWarpBytes;
  int* v = nullptr;
  {
    const cudaError_t e0 = device_once(once, &v, [&](int* val) {
      cudaError_t e = cudaFuncSetAttribute(body_mutate_kernel<MAXD, WARPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
      if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&val[0], body_mutate_kernel<MAXD, WARPS>, WARPS * 32, smem)) != cudaSuccess) return e;
      if (val[0] < 1) val[0] = 1;
      return cudaSuccess;
    });
    if (e0 != cudaSuccess) return e0;
  }
  const int bps = v[0];
  long long want = ((long long)P.n + WARPS - 1) / WARPS, grid = (long long)sm_count * bps;
  if (want < grid) grid = want;
  if (grid < 1) grid = 1;
  body_mutate_kernel<MAXD, WARPS><<<(unsigned)grid, WARPS * 32, smem, st>>>(P);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_body_mutate(const MutateParams& P, uint32_t max_len, int sm_count, cudaStream_t st) {
  if (P.n == 0) return cudaSuccess;
  if (max_len <= 5120) return launch_cls<5120, 4>(P, sm_count, st);
  if (max_len <= 17408) return launch_cls<17408, 2>(P, sm_count, st);
  return launch_cls<65536, 1>(P, sm_count, st);
}

}  // namespace aigw
