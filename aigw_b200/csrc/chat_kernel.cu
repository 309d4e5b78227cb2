// Index (K1), sort (Ks) and emit (K3) stages of the chat translate pass + the launcher.  See chat_kernel.cuh for the design;
// the schema walk (K2) is in chat_walk.cu.  sm_90a only.
//
//   * tokens carry their byte (tty) and a precomputed key / value id (tkid) that 32 lanes compute in
//     parallel, so the schema walk compares one byte instead of strings;
//   * the index stage reads request bodies straight from global memory (the next body is prefetched into L2),
//     so a warp's shared memory holds only its token words; the emit stage stages the body into shared memory
//     by a 1-D bulk asynchronous copy (bulk.cuh) that overlaps the loading of its ops;
//   * the output record is assembled as 16-byte chunks (one chunk per lane, funnel-shifted unaligned
//     reads from shared memory) and stored straight to the arena — no shared-memory image of the output.
#include "chat_internal.cuh"

#include <cstdlib>
#include <mutex>

#include "bulk.cuh"
#include "chat_stage.cuh"

namespace aigw {


// ------------------------------------------------------------------ the kernels
// Launch sequence per sub-batch of documents, intermediates in a reusable global workspace:
//   K1 index   (warp per document)    stage 1+2+2.5 → token words, token count, histogram of token counts
//   Ks sort    (tiny)                 counting sort of the documents by token count → permutation
//   K2 walk    (thread per document)  stage 3+4 → jump table, copy ops, scratch, plan header
//   K3 emit    (warp per document)    stage 5 → output record + result
// K2 is where SIMT pays: 32 bodies with the same token count (≈ the same shape) share every instruction fetch.
// A call of several sub-batches runs K1 of sub-batch k+1 and K3 of sub-batch k in one paired launch (chat_pair_kernel,
// launch_cls), so the two stages, both latency-bound at the residency their shared memory allows (DESIGN.md §4.1), share the SMs.
// ---- K1: structural index, one warp per document
template <int MAXD>
struct IndexSmem {
  using C = Cls<MAXD>;
  static constexpr int kNcBytes = ((MAXD / 1024 + 1) * 4 + 15) & ~15;   // one word per round: lanes (32-byte blocks) that hold a valid escape the encoder rewrites
  static constexpr int kWarpBytes = C::kTok * 6 + kNcBytes;
};

// the key / value id tables of the request or response schema P.schema names
__device__ __forceinline__ const IdTables* id_tables_of(int schema) {
  return (schema & AIGW_SCHEMA_RERANK) ? &c_ids_rr : (schema & AIGW_SCHEMA_COMPLETIONS) ? &c_ids_cp : (schema & AIGW_SCHEMA_RESPONSES) ? &c_ids_rq : (schema & AIGW_SCHEMA_MESSAGES) ? &c_ids_msg : (schema & 48) == AIGW_SCHEMA_RESP_AWS_BEDROCK ? &c_ids_resp : &c_ids;
}

// The warp indexes documents of the sub-batch [doc0, doc0 + ndocs) (workspace work) until the sub-batch's index counter runs out.
// wb: the warp's shared memory (IndexSmem layout).
template <int MAXD>
__device__ __forceinline__ void index_docs(const ChatParams& P, uint32_t doc0, uint32_t ndocs, uint8_t* work, uint8_t* wb, const IdTables* s_ids, int lane) {
  using C = Cls<MAXD>;
  const WorkPtrs wp = carve(work, ndocs, layout_of<MAXD>());   // carved here, so the paired kernel keeps one stage's pointers live at a time
  uint32_t* s_tw = (uint32_t*)wb;
  uint16_t* s_bs = (uint16_t*)(s_tw + C::kTok);   // running backslash count in front of each token; later overlaid by the lookup list
  uint32_t* s_nc = (uint32_t*)(wb + C::kTok * 6);

  // work fetch, one document ahead: the atomic and the location loads of document k+1 complete under the scan of document k
  uint32_t li = 0;
  if (lane == 0) li = atomicAdd(wp.c_index, 1u);
  li = __shfl_sync(FULL, li, 0);
  uint32_t doc = 0, len = 0; const uint8_t* g = nullptr;
  if (li < ndocs) { doc = P.doc_map ? P.doc_map[doc0 + li] : doc0 + li; len = P.lens[doc]; g = P.bodies + P.offsets[doc]; }
  while (li < ndocs) {
    uint32_t li_next = 0;
    if (lane == 0) li_next = atomicAdd(wp.c_index, 1u);
    li_next = __shfl_sync(FULL, li_next, 0);
    uint32_t ndoc = 0, nlen = 0; const uint8_t* ng = nullptr;
    if (li_next < ndocs) { ndoc = P.doc_map ? P.doc_map[doc0 + li_next] : doc0 + li_next; nlen = P.lens[ndoc]; ng = P.bodies + P.offsets[ndoc]; }
#define AIGW_NEXT_DOC() do { li = li_next; doc = ndoc; len = nlen; g = ng; } while (0)
    if (len > (uint32_t)MAXD || len == 0) {
      if (lane == 0) { wp.ntok[li] = 0x80000000u | (len ? AIGW_R_TOO_LARGE : AIGW_R_E400_SYNTAX); atomicAdd(&wp.bins[0], 1u); }
      AIGW_NEXT_DOC();
      continue;
    }
    // the next document starts its way from DRAM to L2 now (its location was loaded under the previous document's scan)
    if (lane == 0 && nlen && nlen <= (uint32_t)MAXD && (reinterpret_cast<uintptr_t>(ng) & 15u) == 0) bulk_prefetch_l2(ng, (nlen + 15u) & ~15u);
    // ---- stages 1 + 2 + 2.5: structural index of the body, read from global memory (chat_stage.cuh)
    const uint32_t ntw = index_doc<MAXD, kBodyGlobal>(g, len, lane, s_tw, s_bs, s_nc, s_ids);
    if (ntw & 0x80000000u) { if (lane == 0) { wp.ntok[li] = ntw; atomicAdd(&wp.bins[0], 1u); } AIGW_NEXT_DOC(); continue; }
    const uint32_t ntok = ntw & 0x3fffffffu;
    // ---- write the token words out, coalesced; histogram of token counts for the shape sort
    {
      uint32_t* gt = wp.tw + (size_t)li * C::kTok;
      for (uint32_t i = lane; i < ntok; i += 32) gt[i] = s_tw[i];
      if (lane == 0) { wp.ntok[li] = ntw; atomicAdd(&wp.bins[bin_of(ntok)], 1u); }
    }
    __syncwarp();
    AIGW_NEXT_DOC();
  }
#undef AIGW_NEXT_DOC
}

// Registers are held to 64 (min_ctas CTAs of WARPS warps = 32 warps per SM), so that the register file is not what caps the
// residency the shared-memory layouts allow.  The 2048 class's index CTAs are small enough for 9 per SM (36 warps, what its staged
// layout had at 56 registers), so its index kernel is held to 56.
template <int WARPS>
__host__ __device__ constexpr int min_ctas() { return 32 / WARPS; }

template <int MAXD, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, MAXD <= 2048 ? 9 : min_ctas<WARPS>()) chat_index_kernel(const __grid_constant__ ChatParams P, uint32_t doc0, uint32_t ndocs, uint8_t* work) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // CTA-shared tables: key/value id hash tables
  IdTables* s_ids = (IdTables*)smem;
  {
    const uint32_t* src = (const uint32_t*)id_tables_of(P.schema);
    for (uint32_t i = threadIdx.x; i < sizeof(IdTables) / 4; i += blockDim.x) ((uint32_t*)s_ids)[i] = src[i];
  }
  __syncthreads();
  index_docs<MAXD>(P, doc0, ndocs, work, smem + sizeof(IdTables) + (size_t)warp * IndexSmem<MAXD>::kWarpBytes, s_ids, lane);
}

// ---- Ks: counting sort by token count (documents with the same count almost always have the same shape).  Every block
// scans the (tiny) histogram itself; positions inside a bin come from a global cursor.  Most documents of a corpus share a few
// bins, so the lanes of a warp that hold the same bin take their positions with ONE atomic (match + rank): one atomic per
// document serialised on those few cursors and made this kernel ~0.1 ms per 229 376 documents on an H100.
__global__ void __launch_bounds__(1024) chat_sort_kernel(const uint32_t* ntok, const uint32_t* bins, uint32_t* cursor, uint32_t* perm, uint32_t ndocs) {
  __shared__ uint32_t s[kBins];
  const int t = threadIdx.x, lane = t & 31;
  const uint32_t v = bins[t];
  s[t] = v;
  __syncthreads();
  for (int off = 1; off < kBins; off <<= 1) { const uint32_t x = t >= off ? s[t - off] : 0u; __syncthreads(); s[t] += x; __syncthreads(); }
  const uint32_t excl = s[t] - v;
  __syncthreads();
  s[t] = excl;
  __syncthreads();
  for (uint32_t l0 = blockIdx.x * blockDim.x; l0 < ndocs; l0 += gridDim.x * blockDim.x) {   // l0 is uniform: every warp runs every round
    const uint32_t li = l0 + t;
    const bool valid = li < ndocs;
    const unsigned act = __ballot_sync(FULL, valid);
    if (!valid) continue;
    const uint32_t b = bin_of(ntok[li]);
    const unsigned peers = __match_any_sync(act, b);
    const int leader = __ffs(peers) - 1;
    uint32_t base = 0;
    if (lane == leader) base = atomicAdd(&cursor[b], (uint32_t)__popc(peers));
    base = __shfl_sync(peers, base, leader);
    perm[s[b] + base + __popc(peers & ((1u << lane) - 1u))] = li;
  }
}

// ---- K3: emit, one warp per document.
// The body is staged by one bulk asynchronous copy while the warp loads the ops and scans their lengths.  Output is built
// as 16-byte chunks, one chunk per lane: the op a chunk starts in comes from a scatter (last op starting at or before each
// chunk) + running max scan instead of a search; chunks inside one op are a single funnel-shifted shared-memory read; the
// chunks that straddle op boundaries are collected and assembled afterwards with every lane busy.
// The warp emits documents of the sub-batch [doc0, doc0 + ndocs) (workspace wp) until the sub-batch's emit counter runs out.
// wb: the warp's shared memory (EmitSmem layout), s_lits: the CTA's copy of the literal table.
template <int MAXD>
__device__ __forceinline__ void emit_docs(const ChatParams& P, uint32_t doc0, uint32_t ndocs, const WorkPtrs& wp, uint8_t* wb, const uint8_t* s_lits, uint64_t* bar, uint32_t& phase, int lane) {
  using C = Cls<MAXD>;
  using E = EmitSmem<MAXD>;
  uint8_t* s_in = wb;
  uint32_t* s_pre = (uint32_t*)(wb + C::kIn);
  uint32_t* s_ops = s_pre + C::kOps + 4;
  uint8_t* s_scr = (uint8_t*)(s_ops + C::kOps);
  uint16_t* s_first = (uint16_t*)(s_scr + E::kScrB);
  uint32_t* s_bl = (uint32_t*)(s_first + kEmitTile);

  // work fetch, one document ahead: plan header, location and the first 32 ops of document k+1 are loaded under the emit of
  // document k (each of these loads used to stall the warp for a DRAM round trip at the top of the loop)
  struct Meta { uint32_t doc, len; const uint8_t* g; PlanOut po; uint32_t op0; };
  auto load_meta = [&](uint32_t l) {
    Meta m;
    m.doc = P.doc_map ? P.doc_map[doc0 + l] : doc0 + l;
    m.len = P.lens[m.doc]; m.g = P.bodies + P.offsets[m.doc];
    m.po = wp.plan[l];
    m.op0 = (wp.ops + (size_t)l * (C::kOps + kSysCap))[lane];
    return m;
  };
  uint32_t li = 0;
  if (lane == 0) li = atomicAdd(wp.c_emit, 1u);
  li = __shfl_sync(FULL, li, 0);
  Meta cur{};
  if (li < ndocs) cur = load_meta(li);
  while (li < ndocs) {
    uint32_t li_next = 0;
    if (lane == 0) li_next = atomicAdd(wp.c_emit, 1u);
    li_next = __shfl_sync(FULL, li_next, 0);
    Meta nxt{};
    if (li_next < ndocs) nxt = load_meta(li_next);
    const uint32_t doc = cur.doc, len = cur.len;
    const PlanOut po = cur.po;
    const uint32_t op_first = cur.op0;
    const uint8_t* g = cur.g;
    aigw_doc_result res = blank_result(len);
    if (po.reason) {
      res.reason = po.reason;
      res.status = po.reason >= 48 ? AIGW_INTERNAL : po.reason >= 40 ? AIGW_INVALID_422 : po.reason >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED;
      if (lane == 0) P.results[doc] = res;
      li = li_next; cur = nxt;
      continue;
    }
    const uint32_t nops = po.nops, olen = po.olen;
    const bool bulk = (reinterpret_cast<uintptr_t>(g) & 15u) == 0;
    if (bulk) { if (lane == 0) { const uint32_t nbytes = (len + 15u) & ~15u; mbar_expect_tx(bar, nbytes); bulk_g2s(s_in, g, nbytes, bar); } }
    else for (uint32_t i = lane; i < len; i += 32) s_in[i] = g[i];
    // while the body is in flight: ops (+ exclusive prefix of their lengths) and the scratch bytes they reference
    const uint32_t scr_hi = emit_prefix<MAXD>(wp.ops + (size_t)li * (C::kOps + kSysCap), op_first, nops, olen, s_ops, s_pre, lane);
    { const uint8_t* gs = wp.scr + (size_t)li * C::kScr; for (uint32_t i = lane; i < ((scr_hi + 3u) >> 2); i += 32) ((uint32_t*)s_scr)[i] = ((const uint32_t*)gs)[i]; }
    const uint32_t rec = (olen + 15u) & ~15u;
    const uint32_t nchunks = rec >> 4;
    unsigned long long obase = 0;
    if (lane == 0) obase = atomicAdd(P.out_used, (unsigned long long)rec);
    obase = __shfl_sync(FULL, obase, 0);
    __syncwarp();
    if (bulk) { mbar_wait(bar, phase); phase ^= 1u; }
    if (obase + rec > P.out_capacity || nchunks > 0xffffu) {
      res.reason = nchunks > 0xffffu ? AIGW_R_OUT_SPACE : AIGW_R_ARENA_FULL;
      if (lane == 0) P.results[doc] = res;
      __syncwarp();
      li = li_next; cur = nxt;
      continue;
    }
    if (lane == 0 && li_next < ndocs && !nxt.po.reason && (reinterpret_cast<uintptr_t>(nxt.g) & 15u) == 0) bulk_prefetch_l2(nxt.g, (nxt.len + 15u) & ~15u);
    uint4* o4 = (uint4*)(P.out + obase);
    emit_doc<MAXD>(s_in, s_lits, s_scr, s_pre, s_ops, s_first, s_bl, nops, nchunks, o4, lane);
    if (lane == 0) {
      res.out_off = obase + P.out_bias; res.body_len = olen - po.path_len; res.path_len = (uint16_t)po.path_len; res.status = AIGW_OK; res.reason = 0;
      res.model_off = po.model_off; res.model_len = po.model_len; res.body_kind = (po.flags & 0x80u) ? AIGW_BODY_UNCHANGED : AIGW_BODY_BYTES; res.flags = po.flags & 0x7fu;
      P.results[doc] = res;
    }
    __syncwarp();
    li = li_next; cur = nxt;
  }
}

template <int MAXD, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) chat_emit_kernel(const __grid_constant__ ChatParams P, uint32_t doc0, uint32_t ndocs, uint8_t* work) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint8_t* s_lits = smem;
  uint64_t* s_bar = (uint64_t*)(smem + sizeof(c_lits.bytes));
  for (uint32_t i = threadIdx.x; i < sizeof(c_lits.bytes) / 4; i += blockDim.x) ((uint32_t*)s_lits)[i] = ((const uint32_t*)c_lits.bytes)[i];
  if (threadIdx.x == 0) { for (int w = 0; w < WARPS; w++) mbar_init(&s_bar[w], 1); mbar_fence_init(); }
  __syncthreads();
  constexpr int kHdr = (int)((sizeof(c_lits.bytes) + 8 * WARPS + 15) & ~(size_t)15);
  uint32_t phase = 0;
  emit_docs<MAXD>(P, doc0, ndocs, carve(work, ndocs, layout_of<MAXD>()), smem + kHdr + (size_t)warp * EmitSmem<MAXD>::kWarpBytes, s_lits, &s_bar[warp], phase, lane);
}

// ---- K1 + K3 paired: the index of sub-batch k+1 and the emit of sub-batch k share the SMs in one launch.  There is no data
// dependency between the two (separate workspace slots), so each CTA holds the header of both (id tables, literal table).  Its
// first EW warps are emit warps: each has an EmitSmem region (the staged body among it) and an mbarrier, starts on the emit list
// and joins the index list when the emit list runs out.  The other IW warps are index warps with an IndexSmem region, which has no
// room for a body: they index until the index list runs out and then exit.  An index warp's region is a third to a half of an emit
// warp's, so an SM keeps more warps resident than with CTAs of union-sized regions.  With IW = 0 every warp has an emit region
// (the union of the two layouts), even warps start on the index list and odd warps on the emit list, and a warp that drains its
// list joins the other one: the layout for classes where the split gains no residency.
template <int EW>
__host__ __device__ constexpr size_t pair_hdr_bytes() { return (sizeof(IdTables) + sizeof(LitTable::bytes) + 8 * EW + 15) & ~(size_t)15; }
template <int MAXD, int EW, int IW>
__host__ __device__ constexpr size_t pair_smem_bytes() { return pair_hdr_bytes<EW>() + (size_t)EmitSmem<MAXD>::kWarpBytes * EW + (size_t)IndexSmem<MAXD>::kWarpBytes * IW; }
// an emit warp indexes in its own region once the emit list runs out
static_assert(EmitSmem<2048>::kWarpBytes >= IndexSmem<2048>::kWarpBytes && EmitSmem<5120>::kWarpBytes >= IndexSmem<5120>::kWarpBytes &&
              EmitSmem<9216>::kWarpBytes >= IndexSmem<9216>::kWarpBytes && EmitSmem<17408>::kWarpBytes >= IndexSmem<17408>::kWarpBytes &&
              EmitSmem<33792>::kWarpBytes >= IndexSmem<33792>::kWarpBytes && EmitSmem<65536>::kWarpBytes >= IndexSmem<65536>::kWarpBytes,
              "an emit warp's region must hold the index layout");

template <int MAXD, int EW, int IW>
__global__ void __launch_bounds__((EW + IW) * 32, min_ctas<EW + IW>()) chat_pair_kernel(const __grid_constant__ ChatParams P, uint32_t doc0_idx, uint32_t n_idx, uint8_t* work_idx,
                                                                                        uint32_t doc0_emit, uint32_t n_emit, uint8_t* work_emit) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  IdTables* s_ids = (IdTables*)smem;
  uint8_t* s_lits = smem + sizeof(IdTables);
  uint64_t* s_bar = (uint64_t*)(s_lits + sizeof(c_lits.bytes));
  {
    const uint32_t* src = (const uint32_t*)id_tables_of(P.schema);
    for (uint32_t i = threadIdx.x; i < sizeof(IdTables) / 4; i += blockDim.x) ((uint32_t*)s_ids)[i] = src[i];
    for (uint32_t i = threadIdx.x; i < sizeof(c_lits.bytes) / 4; i += blockDim.x) ((uint32_t*)s_lits)[i] = ((const uint32_t*)c_lits.bytes)[i];
  }
  if (threadIdx.x == 0) { for (int w = 0; w < EW; w++) mbar_init(&s_bar[w], 1); mbar_fence_init(); }
  __syncthreads();
  uint8_t* regions = smem + pair_hdr_bytes<EW>();
  if constexpr (IW == 0) {
    uint8_t* wb = regions + (size_t)warp * EmitSmem<MAXD>::kWarpBytes;
    uint32_t phase = 0;
    if ((warp & 1) == 0) {
      index_docs<MAXD>(P, doc0_idx, n_idx, work_idx, wb, s_ids, lane);
      emit_docs<MAXD>(P, doc0_emit, n_emit, carve(work_emit, n_emit, layout_of<MAXD>()), wb, s_lits, &s_bar[warp], phase, lane);
    } else {
      emit_docs<MAXD>(P, doc0_emit, n_emit, carve(work_emit, n_emit, layout_of<MAXD>()), wb, s_lits, &s_bar[warp], phase, lane);
      index_docs<MAXD>(P, doc0_idx, n_idx, work_idx, wb, s_ids, lane);
    }
  } else if (warp < EW) {
    uint8_t* wb = regions + (size_t)warp * EmitSmem<MAXD>::kWarpBytes;
    uint32_t phase = 0;
    emit_docs<MAXD>(P, doc0_emit, n_emit, carve(work_emit, n_emit, layout_of<MAXD>()), wb, s_lits, &s_bar[warp], phase, lane);
    index_docs<MAXD>(P, doc0_idx, n_idx, work_idx, wb, s_ids, lane);
  } else {
    index_docs<MAXD>(P, doc0_idx, n_idx, work_idx, regions + (size_t)EW * EmitSmem<MAXD>::kWarpBytes + (size_t)(warp - EW) * IndexSmem<MAXD>::kWarpBytes, s_ids, lane);
  }
}

// ------------------------------------------------------------------ host-side launcher
template <int MAXD>
size_t work_bytes_cls(size_t ndocs) { return work_per_doc(layout_of<MAXD>()) * ndocs + kWorkHdr + 256; }

struct ClsConfig { bool ready = false; int bps1 = 1, bps3 = 1, bpsp = 1; };

// Paired schedule (launch_cls): documents per sub-batch, at most; two workspace slots of this size must fit the 3 GiB workspace
// cap (lib.cu ensure_chat_work), which a slot of more than ~236 000 documents at the 5120 class does not.  Every sub-batch adds a
// walk launch with its own tail, and that costs more than the pairing saves at smaller sizes.  Measured on an H100 80GB HBM3 at
// 700 W (SM 1980 MHz, no throttle), bench.py's config-2 call (1 M bodies of ~4 KB), paired vs the serial schedule in one process
// (tools/bench_translate_schedule.py): 65 536: 14.57 vs 12.07 ms; 131 072: 11.84 vs 11.76 ms; 229 376: 11.62 vs 11.77 ms.
// A call pairs only when it holds at least two full sub-batches of this size (kPairMinSubBatches; the workspace cap may then cut
// the sub-batch of a large class smaller): below that the serial schedule runs it in one or two sub-batches of up to 262 144
// documents.  The host call's chunks of ~1 KB bodies (bench.py config 5), paired at 131 072, were 7 % slower.  The call is
// then cut into equal sub-batches of at most this size.  AIGW_CHAT_SUB overrides the size for measurements.
static constexpr size_t kPairSubDocs = 229376;
static constexpr size_t kPairMinSubBatches = 2;
static size_t pair_sub_docs() {
  static const long env = getenv("AIGW_CHAT_SUB") ? atol(getenv("AIGW_CHAT_SUB")) : 0;
  return env > 0 ? (size_t)env : kPairSubDocs;
}

// Emit and index warps per CTA of the paired kernel, per class (H100: 228 KB of shared memory per SM, 1 KB reserved per CTA; the CTA
// header is 8 448 bytes of tables + one mbarrier per emit warp; see DESIGN.md §4.1 for the per-warp regions):
//   class   emit + index warps / CTA   CTAs x warps / SM    shared memory / CTA
//   2048     8 + 0                      4 x 8  = 32          54 976 B
//   5120     6 + 10                     2 x 16 = 32         109 712 B
//   9216     4 + 4                      2 x 8  = 16         102 560 B
//   17408    2 + 3                      2 x 5  = 10         105 568 B
// At 2048 the pair is held to 4 CTAs by its 64 registers, not by shared memory, so a split would gain no warps and only take the
// emit list away from half of them: every warp keeps the union region.  Paired calls of 459 752 bodies timed against the union
// layout (DESIGN.md §4.1): 9216 5.78-5.83 vs 6.44-6.47 ms, 17408 8.16-8.19 vs 10.74-10.75 ms.
// 0: the class keeps the serial schedule.  At 33792 and 65536 an emit warp's region alone is 53 424 and 101 040 B, so a paired CTA
// of one emit and one index warp keeps fewer emit warps on an SM than the serial emit kernel does (2 vs 4 and 1 vs 2).
constexpr int pair_emit_warps(int maxd) { return maxd <= 2048 ? 8 : maxd <= 5120 ? 6 : maxd <= 9216 ? 4 : maxd <= 17408 ? 2 : 0; }
constexpr int pair_index_warps(int maxd) { return maxd <= 2048 ? 0 : maxd <= 5120 ? 10 : maxd <= 9216 ? 4 : maxd <= 17408 ? 3 : 0; }
static int class_of(uint32_t max_len) { return max_len <= 2048 ? 2048 : max_len <= 5120 ? 5120 : max_len <= 9216 ? 9216 : max_len <= 17408 ? 17408 : max_len <= 33792 ? 33792 : 65536; }
// one slot of the paired schedule: `sub` documents' intermediates, 256-byte aligned
static size_t pair_slot_bytes(int maxd, size_t sub) { return (chat_work_bytes((uint32_t)maxd, sub) + 255) & ~(size_t)255; }

// WI / WE: warps per CTA of the serial index / emit kernel
template <int MAXD, int WI, int WE>
static cudaError_t launch_cls(const ChatParams& P, uint32_t first, int device, int sm_count, cudaStream_t st, uint8_t* work, size_t work_cap, cudaEvent_t* ev, int ev_cap,
                              int* launches) {
  using C = Cls<MAXD>;
  constexpr bool kPair = pair_emit_warps(MAXD) > 0;
  constexpr int EW = kPair ? pair_emit_warps(MAXD) : 1, IW = kPair ? pair_index_warps(MAXD) : 1, PW = EW + IW;   // used when kPair
  constexpr size_t hdr1 = sizeof(IdTables), hdr3 = (sizeof(LitTable::bytes) + 8 * WE + 15) & ~(size_t)15;
  const size_t smem1 = hdr1 + (size_t)IndexSmem<MAXD>::kWarpBytes * WI;
  const size_t smem3 = hdr3 + (size_t)EmitSmem<MAXD>::kWarpBytes * WE;
  constexpr size_t smemp = pair_smem_bytes<MAXD, EW, IW>();
  static_assert(smemp <= 227 * 1024, "paired kernel's shared memory exceeds a CTA's limit");
  static ClsConfig cfgs[kMaxDevices];
  static std::mutex mu;
  if (device < 0 || device >= kMaxDevices) return cudaErrorInvalidDevice;
  ClsConfig& cc = cfgs[device];
  {
    std::lock_guard<std::mutex> lk(mu);
    if (!cc.ready) {
      cudaError_t e = cudaFuncSetAttribute(chat_index_kernel<MAXD, WI>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1);
      if (e != cudaSuccess) return e;
      e = cudaFuncSetAttribute(chat_emit_kernel<MAXD, WE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem3);
      if (e != cudaSuccess) return e;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cc.bps1, chat_index_kernel<MAXD, WI>, WI * 32, smem1);
      if (e != cudaSuccess) return e;
      e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cc.bps3, chat_emit_kernel<MAXD, WE>, WE * 32, smem3);
      if (e != cudaSuccess) return e;
      if constexpr (kPair) {
        e = cudaFuncSetAttribute(chat_pair_kernel<MAXD, EW, IW>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smemp);
        if (e != cudaSuccess) return e;
        e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cc.bpsp, chat_pair_kernel<MAXD, EW, IW>, PW * 32, smemp);
        if (e != cudaSuccess) return e;
      }
      if (cc.bps1 < 1) cc.bps1 = 1;
      if (cc.bps3 < 1) cc.bps3 = 1;
      if (cc.bpsp < 1) cc.bpsp = 1;
      cc.ready = true;
    }
  }
  // ---- paired schedule, two workspace slots (sub-batch k in slot k mod 2), one stream:
  //   I(0) · S(0) W(0) · P(I(1)+E(0)) · S(1) W(1) · P(I(2)+E(1)) · … · S(n−1) W(n−1) · E(n−1)
  // P is chat_pair_kernel: the index of the next sub-batch and the emit of this one share the SMs.  The walk runs alone (its
  // registers make the register file the binding resource when it shares an SM).  Stage timing (ev) keeps the serial schedule
  // below, whose four launches per sub-batch are what the stage split is read from.
  if constexpr (kPair) {
    const size_t slot = (work_cap / 2) & ~(size_t)255;
    size_t sub = slot > (size_t)kWorkHdr + 256 ? (slot - kWorkHdr - 256) / work_per_doc(layout_of<MAXD>()) : 0;
    if (sub > pair_sub_docs()) sub = pair_sub_docs();
    if (!ev && sub > 0 && P.n >= kPairMinSubBatches * pair_sub_docs()) {
      // equal sub-batches: a short last one would add a walk launch whose tail is as long as a full one's
      const uint32_t nsb = (uint32_t)((P.n + sub - 1) / sub);
      sub = (P.n + nsb - 1) / nsb;
      auto nd_of = [&](uint32_t k) { return (uint32_t)((size_t)P.n - (size_t)k * sub < sub ? (size_t)P.n - (size_t)k * sub : sub); };
      auto wk_of = [&](uint32_t k) { return work + (size_t)(k & 1u) * slot; };
      auto grid = [&](long long units, int warps, int bps) { long long g = (long long)sm_count * bps, want = (units + warps - 1) / warps; return (unsigned)(want < g ? want : g); };
      cudaError_t e;
      if ((e = cudaMemsetAsync(wk_of(0), 0, kWorkHdr, st)) != cudaSuccess) return e;
      chat_index_kernel<MAXD, WI><<<grid(nd_of(0), WI, cc.bps1), WI * 32, smem1, st>>>(P, first, nd_of(0), wk_of(0));
      int nl = 1;
      for (uint32_t k = 0; k < nsb; k++) {
        const uint32_t nd = nd_of(k), doc0 = first + (uint32_t)(k * sub);
        uint8_t* wk = wk_of(k);
        const WorkPtrs wp = carve(wk, nd, layout_of<MAXD>());
        { const unsigned gs = (nd + 8191) / 8192; chat_sort_kernel<<<gs < 32 ? gs : 32, kBins, 0, st>>>(wp.ntok, wp.bins, wp.cursor, wp.perm, nd); }
        if ((e = launch_chat_walk(P, doc0, nd, wk, layout_of<MAXD>(), st, sm_count)) != cudaSuccess) return e;
        if (k + 1 < nsb) {
          // slot (k+1) mod 2 was last used by sub-batch k-1, whose emit ran in the previous paired launch
          const uint32_t nn = nd_of(k + 1);
          if ((e = cudaMemsetAsync(wk_of(k + 1), 0, kWorkHdr, st)) != cudaSuccess) return e;
          chat_pair_kernel<MAXD, EW, IW><<<grid((long long)nn + nd, PW, cc.bpsp), PW * 32, smemp, st>>>(P, doc0 + nd, nn, wk_of(k + 1), doc0, nd, wk);
        } else {
          chat_emit_kernel<MAXD, WE><<<grid(nd, WE, cc.bps3), WE * 32, smem3, st>>>(P, doc0, nd, wk);
        }
        nl += 3;
      }
      if (launches) *launches = nl;
      return cudaGetLastError();
    }
  }
  // ---- serial schedule, one stream, the whole workspace: index · sort · walk · emit per sub-batch of up to 262 144 documents
  size_t sub = ((work_cap & ~(size_t)255) - kWorkHdr - 256) / work_per_doc(layout_of<MAXD>());
  if (sub > 262144) sub = 262144;
  if (sub == 0) return cudaErrorMemoryAllocation;
  cudaError_t e;
  int nl = 0, sb = 0;
  for (uint32_t rel = 0; rel < P.n; rel += (uint32_t)sub, sb++) {
    const uint32_t doc0 = first + rel;
    const uint32_t nd = (uint32_t)(P.n - rel < sub ? P.n - rel : sub);
    const WorkPtrs wp = carve(work, nd, layout_of<MAXD>());
    if ((e = cudaMemsetAsync(work, 0, kWorkHdr, st)) != cudaSuccess) return e;
    long long g1 = (long long)sm_count * cc.bps1; if (((long long)nd + WI - 1) / WI < g1) g1 = ((long long)nd + WI - 1) / WI;
    long long g3 = (long long)sm_count * cc.bps3; if (((long long)nd + WE - 1) / WE < g3) g3 = ((long long)nd + WE - 1) / WE;
    const bool timed = ev && 4 * sb + 3 < ev_cap;
    if (timed) cudaEventRecord(ev[4 * sb + 0], st);
    chat_index_kernel<MAXD, WI><<<(unsigned)g1, WI * 32, smem1, st>>>(P, doc0, nd, work);
    if (timed) cudaEventRecord(ev[4 * sb + 1], st);
    { const unsigned gs = (nd + 8191) / 8192; chat_sort_kernel<<<gs < 32 ? gs : 32, kBins, 0, st>>>(wp.ntok, wp.bins, wp.cursor, wp.perm, nd); }
    if ((e = launch_chat_walk(P, doc0, nd, work, layout_of<MAXD>(), st, sm_count)) != cudaSuccess) return e;
    if (timed) cudaEventRecord(ev[4 * sb + 2], st);
    chat_emit_kernel<MAXD, WE><<<(unsigned)g3, WE * 32, smem3, st>>>(P, doc0, nd, work);
    if (timed) cudaEventRecord(ev[4 * sb + 3], st);
    nl += 4;
  }
  if (launches) *launches = nl;
  return cudaGetLastError();
}

size_t chat_work_bytes(uint32_t max_len, size_t ndocs) {
  if (max_len <= 2048) return work_bytes_cls<2048>(ndocs);
  if (max_len <= 5120) return work_bytes_cls<5120>(ndocs);
  if (max_len <= 9216) return work_bytes_cls<9216>(ndocs);
  if (max_len <= 17408) return work_bytes_cls<17408>(ndocs);
  if (max_len <= 33792) return work_bytes_cls<33792>(ndocs);
  return work_bytes_cls<65536>(ndocs);
}
// workspace that lets a call of n documents run its schedule: two slots of the paired schedule, or one sub-batch
size_t chat_work_bytes_for(uint32_t max_len, size_t n) {
  const int maxd = class_of(max_len);
  if (pair_emit_warps(maxd) > 0 && n >= kPairMinSubBatches * pair_sub_docs()) return 2 * pair_slot_bytes(maxd, pair_sub_docs()) + 512;
  return chat_work_bytes(max_len, n < 262144 ? n : 262144) + 512;
}

cudaError_t launch_chat_translate(const ChatParams& P, uint32_t max_len, int device, int sm_count, cudaStream_t st, uint8_t* work, size_t work_cap, int* launches,
                                  cudaEvent_t* ev, int ev_cap, uint32_t first) {
  if (max_len <= 2048) return launch_cls<2048, 4, 4>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
  if (max_len <= 5120) return launch_cls<5120, 4, 4>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
  if (max_len <= 9216) return launch_cls<9216, 4, 2>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
  if (max_len <= 17408) return launch_cls<17408, 2, 2>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
  if (max_len <= 33792) return launch_cls<33792, 2, 1>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
  return launch_cls<65536, 1, 1>(P, first, device, sm_count, st, work, work_cap, ev, ev_cap, launches);
}

}  // namespace aigw
