// K4: byte-level BPE token count on the GPU (north_star: "a GPU BPE tokenizer with the merge table staged in shared memory for
// token-based rate limiting").  The reference has no tokenizer (SURVEY F4), so the semantics are the ones include/aigw_b200.h
// states and tests/golden/make_bpe_vocab.py fixes with HuggingFace `tokenizers`:
//   pre-tokenisation  every space starts a new piece; a piece is its first byte plus the bytes up to the next space
//   model             inside a piece, merge the adjacent pair of lowest rank (leftmost first among equal ranks) until none is mergeable
//   result            tokens per text = sum of the pieces' final lengths
//
// Mapping.  Persistent CTAs; the merge table (open-addressing hash, key = a << 16 | b, value = rank << 16 | merged) is copied into
// shared memory once per CTA.  A warp pulls a GROUP of consecutive texts whose bytes fit its staging buffer (short inputs — 64
// characters in BASELINE config 3 — would leave most lanes idle one text at a time), stages the bytes, turns
// them into symbol ids, finds the piece starts with ballots, and then every LANE runs the merge loop of one piece at a time
// (pieces are independent).  Per piece the ranks of the adjacent pairs are kept next to the symbols, so a merge costs two
// table lookups and one shift instead of a rescan.  A text longer than the buffer is cut at piece boundaries; a single piece
// longer than the buffer is DECLINED (count 0xFFFFFFFF) rather than approximated.  sm_90a only.
#include "bpe_kernel.cuh"

#include <cstdio>

namespace aigw {

static constexpr int kBpeWarps = 32;            // the merge loops are latency-bound (dependent shared-memory lookups): as many warps as shared memory allows
static constexpr int kBpeBuf = 512;            // staged bytes per warp (a piece longer than this is declined); small, so that 32 warps fit beside the table
static constexpr int kBpeMaxTexts = 32;         // texts per group
static constexpr uint32_t kEmpty = 0xffffffffu;

__device__ __forceinline__ uint32_t bpe_hash(uint32_t key) { key *= 0x9E3779B1u; return key ^ (key >> 15); }

// rank << 16 | merged of the pair (a, b), or kEmpty
__device__ __forceinline__ uint32_t bpe_lookup(const uint2* tab, uint32_t mask, uint32_t a, uint32_t b) {
  const uint32_t key = (a << 16) | b;
  uint32_t s = bpe_hash(key) & mask;
  for (;;) {
    const uint2 e = tab[s];
    if (e.x == key) return e.y;
    if (e.x == kEmpty) return kEmpty;
    s = (s + 1) & mask;
  }
}

struct BpeWarpSmem {
  uint8_t bytes[kBpeBuf + 16];
  uint32_t sr[kBpeBuf];          // symbol | rank << 16 of the pair (this symbol, next live symbol); rank 0xffff = not mergeable, 0xfffe = slot merged away
  uint16_t start[kBpeBuf + 1];   // piece starts, ascending; start[np] = end of data
  uint32_t stmask[kBpeBuf / 32 + 1];   // bit i of word b: byte 32 b + i starts a piece
  uint32_t next_piece;           // pieces handed out so far in this run (lanes take the next one when theirs is done)
  uint32_t tcount[kBpeMaxTexts];
  uint32_t tend[kBpeMaxTexts];   // staged end offset of each text of the group
};

__global__ void __launch_bounds__(kBpeWarps * 32, 1) bpe_count_kernel(const BpeParams P) {
  extern __shared__ __align__(16) uint8_t smem[];
  uint2* tab = (uint2*)smem;
  const uint32_t mask = P.slots - 1u;
  for (uint32_t i = threadIdx.x; i < P.slots; i += blockDim.x) tab[i] = P.table[i];
  __shared__ uint16_t s_b2i[256];
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) s_b2i[i] = P.byte_to_id[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  BpeWarpSmem& W = *(BpeWarpSmem*)(smem + (size_t)P.slots * 8 + (size_t)warp * sizeof(BpeWarpSmem));

  for (;;) {
    // ---- a group of consecutive texts: the counter hands out kBpeMaxTexts at a time, the warp walks them in buffer-sized runs
    uint32_t g0 = 0;
    if (lane == 0) g0 = atomicAdd(P.next, (unsigned)kBpeMaxTexts);
    g0 = __shfl_sync(0xffffffffu, g0, 0);
    if (g0 >= P.n) break;
    const uint32_t g1 = min(P.n, g0 + (uint32_t)kBpeMaxTexts);
    uint32_t t = g0;        // next text to stage
    uint32_t t_off = 0;     // bytes of text t already counted (a text longer than the buffer is cut at piece boundaries)
    uint32_t t_acc = 0;     // tokens of that counted part
    while (t < g1) {
      // ---- stage texts t, t+1, … while they fit
      const uint32_t first = t; const bool first_cont = t_off != 0;
      uint32_t fill = 0, nt = 0; bool last_partial = false;
      while (t < g1) {
        const uint32_t len = P.lens[t] - t_off;
        const uint8_t* src = P.text + P.offsets[t] + t_off;
        uint32_t take = len;
        if (fill + len > (uint32_t)kBpeBuf) {
          if (nt > 0) break;                                   // what is staged so far is counted first
          uint32_t cut = 0;                                    // the last piece start inside the window
          for (uint32_t b0 = 0; b0 < (uint32_t)kBpeBuf; b0 += 32) { const uint32_t i = b0 + lane; const uint32_t m = __ballot_sync(0xffffffffu, i > 0 && src[i] == ' '); if (m) cut = b0 + 31u - __clz(m); }
          if (cut == 0) { if (lane == 0) P.counts[t] = 0xffffffffu; t++; t_off = 0; t_acc = 0; break; }   // one piece longer than the buffer: declined
          take = cut; last_partial = true;
        }
        for (uint32_t i = lane; i < take; i += 32) W.bytes[fill + i] = src[i];
        fill += take;
        if (lane == 0) { W.tend[nt] = fill; W.tcount[nt] = 0; }
        nt++;
        if (last_partial) { t_off += take; break; }
        t++; t_off = 0;
      }
      if (nt == 0) continue;
      __syncwarp();
      // ---- symbols and piece starts: a piece starts at every space and at the first byte of every staged text
      for (uint32_t i = lane; i < fill; i += 32) W.sr[i] = 0;
      __syncwarp();
      for (uint32_t k = lane; k < nt; k += 32) { const uint32_t s0 = k == 0 ? 0u : W.tend[k - 1]; if (s0 < fill) W.sr[s0] = 1; }
      __syncwarp();
      uint32_t np = 0;
      for (uint32_t b0 = 0; b0 < fill; b0 += 32) {
        const uint32_t i = b0 + lane;
        const uint32_t c = i < fill ? W.bytes[i] : 0u;
        const bool st = i < fill && (c == ' ' || W.sr[i] != 0);   // the text-start flag is read before the slot takes the symbol
        if (i < fill) W.sr[i] = s_b2i[c];
        const uint32_t m = __ballot_sync(0xffffffffu, st);
        if (st) W.start[np + __popc(m & lt)] = (uint16_t)i;
        if (lane == 0) W.stmask[b0 >> 5] = m;
        np += __popc(m);
      }
      if (lane == 0) { W.start[np] = (uint16_t)fill; W.stmask[(fill + 31) >> 5] = 0xffffffffu; W.next_piece = 0; }
      __syncwarp();
      // ---- ranks of all adjacent pairs, one lane per byte position (a pair never spans two pieces)
      for (uint32_t b0 = 0; b0 < fill; b0 += 32) {
        const uint32_t i = b0 + lane;
        if (i < fill) {
          const uint32_t nx = i + 1;
          const bool last = nx >= fill || ((W.stmask[nx >> 5] >> (nx & 31u)) & 1u);
          const uint32_t sy = W.sr[i] & 0xffffu;
          uint32_t rk = 0xffff0000u;
          if (!last) { const uint32_t v = bpe_lookup(tab, mask, sy, W.sr[nx] & 0xffffu); if (v != kEmpty) rk = v & 0xffff0000u; }
          W.sr[i] = sy | rk;
        }
      }
      __syncwarp();
      // ---- merges: every lane works on one piece and takes the next unclaimed one when it is done, so the lanes stay busy
      // whatever the piece lengths are (one piece per lane per round left 10 of 32 lanes active on average)
      {
        uint32_t a = 0, L0 = 0, L = 0; uint32_t* q = W.sr; bool have = false, done = false;
        for (;;) {
          if (!have && !done) {
            const uint32_t pi = atomicAdd(&W.next_piece, 1u);
            if (pi >= np) done = true;
            else { a = W.start[pi]; L0 = W.start[pi + 1] - a; L = L0; q = W.sr + a; have = true; }
          }
          if (__all_sync(0xffffffffu, done)) break;
          if (have) {
            uint32_t best = 0xfffeu, at = 0;
            if (L > 1) for (uint32_t k = 0; k < L0; k++) { const uint32_t r = q[k] >> 16; if (r < best) { best = r; at = k; } }   // leftmost lowest rank; 0xfffe (merged away) / 0xffff never win
            if (best == 0xfffeu) {   // nothing left to merge: the piece is worth L tokens
              uint32_t lo = 0; while (W.tend[lo] <= a) lo++;      // the text this piece belongs to (empty texts own no piece)
              atomicAdd(&W.tcount[lo], L);
              have = false;
            } else {
              uint32_t j = at + 1; while ((q[j] >> 16) == 0xfffeu) j++;              // the right partner (a mergeable pair has one)
              const uint32_t merged = bpe_lookup(tab, mask, q[at] & 0xffffu, q[j] & 0xffffu) & 0xffffu;
              q[j] = 0xfffe0000u;
              uint32_t rank_at = 0xffffu;
              uint32_t j2 = j + 1; while (j2 < L0 && (q[j2] >> 16) == 0xfffeu) j2++;   // the merged symbol's new right neighbour, if any
              if (j2 < L0) { const uint32_t v = bpe_lookup(tab, mask, merged, q[j2] & 0xffffu); if (v != kEmpty) rank_at = v >> 16; }
              q[at] = merged | (rank_at << 16);
              if (at > 0) {
                uint32_t i = at - 1; bool live = true;
                while ((q[i] >> 16) == 0xfffeu) { if (i == 0) { live = false; break; } i--; }
                if (live) { const uint32_t v = bpe_lookup(tab, mask, q[i] & 0xffffu, merged); q[i] = (q[i] & 0xffffu) | (v == kEmpty ? 0xffff0000u : (v & 0xffff0000u)); }
              }
              L--;
            }
          }
        }
      }
      __syncwarp();
      // ---- results of the texts that ended in this run; a cut text carries its partial count into the next run
      uint32_t carry = 0;
      for (uint32_t k0 = 0; k0 < nt; k0 += 32) {
        const uint32_t k = k0 + lane;
        if (k < nt) {
          const uint32_t c = W.tcount[k] + ((k == 0 && first_cont) ? t_acc : 0u);
          if (k == nt - 1 && last_partial) carry = c; else P.counts[first + k] = c;
        }
      }
      carry = __reduce_max_sync(0xffffffffu, carry);
      t_acc = last_partial ? carry : 0u;
      __syncwarp();
    }
  }
}

size_t bpe_smem_bytes(uint32_t slots) { return (size_t)slots * 8 + (size_t)kBpeWarps * sizeof(BpeWarpSmem); }

cudaError_t launch_bpe_count(const BpeParams& P, int sm_count, cudaStream_t st) {
  const size_t smem = bpe_smem_bytes(P.slots);
  static DeviceOnce once;
  int* vals = nullptr;
  cudaError_t e = device_once(once, &vals, [&](int*) { return cudaFuncSetAttribute(bpe_count_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024); });
  if (e != cudaSuccess) return e;
  if (smem > 220 * 1024) return cudaErrorInvalidValue;
  const unsigned groups = (P.n + kBpeMaxTexts - 1) / kBpeMaxTexts;
  const unsigned want = (groups + kBpeWarps - 1) / kBpeWarps;
  const unsigned grid = want < (unsigned)sm_count ? (want ? want : 1u) : (unsigned)sm_count;
  bpe_count_kernel<<<grid, kBpeWarps * 32, smem, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
