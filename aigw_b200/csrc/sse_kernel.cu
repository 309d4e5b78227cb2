// See sse_kernel.cuh.  sm_90a only.
#include <cstring>
#include <vector>

#include "device_once.cuh"
#include "sse_kernel.cuh"
#include "sse_schema.cuh"

namespace aigw {

__device__ SchemaBlob g_schema;

// ------------------------------------------------------------------ kernel
__device__ __forceinline__ uint32_t nib_ff(uint32_t m) { return ((m & 0x08040201u) * 0x01010101u) >> 24; }   // 0xFF per byte → 4-bit mask
static constexpr int kTile = 8192;       // bytes of a stream staged per warp
static constexpr int kMaxLines = 512;    // line-start slots per tile
static constexpr int kWarps = 4;
static constexpr int kMaxCand = 64;
static constexpr int kWarpBytes = kTile + 32 + kMaxLines * 2 + kMaxLines / 8 + kMaxCand * 2;

struct LineOut { uint32_t seq; uint32_t v[6]; uint32_t flags; uint32_t model_off, model_len; };

__global__ void __launch_bounds__(kWarps * 32) sse_usage_kernel(const __grid_constant__ SseParams P) {
  extern __shared__ __align__(16) uint8_t smem[];
  SchemaBlob* sch = (SchemaBlob*)smem;
  for (uint32_t i = threadIdx.x; i < sizeof(SchemaBlob) / 4; i += blockDim.x) ((uint32_t*)sch)[i] = ((const uint32_t*)&g_schema)[i];
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t FULLM = 0xffffffffu;
  uint8_t* tile = smem + ((sizeof(SchemaBlob) + 15) & ~15u) + (size_t)warp * kWarpBytes;
  uint16_t* lstart = (uint16_t*)(tile + kTile + 32);
  uint32_t* s_need = (uint32_t*)(lstart + kMaxLines);   // bit per line: the typed walk is needed
  uint16_t* s_cand = (uint16_t*)(s_need + kMaxLines / 32);   // positions of `"usage"` / `\u` candidates of the tile

  for (;;) {
    uint32_t s = 0;
    if (lane == 0) s = atomicAdd(P.next, 1u);
    s = __shfl_sync(FULLM, s, 0);
    if (s >= P.n_streams) break;
    const uint64_t sb = P.chunk_off[P.chunk_first[s]], se = P.chunk_off[P.chunk_first[s + 1]];
    // per-lane "latest" records, by group: 0 usage(in/out/total) 1 ptd(cached, creation) 2 ctd(reasoning) 3 model
    uint32_t seq_u = 0, seq_p = 0, seq_c = 0, seq_m = 0;  // 0 = none; line ordinal + 1
    uint32_t v_in = 0, v_out = 0, v_tot = 0, v_cached = 0, v_cc = 0, v_reason = 0;
    uint64_t m_off = 0; uint32_t m_len = 0;
    uint32_t status = 0;
    uint32_t line_no = 0;
    uint64_t pos = sb;         // next unread stream byte
    uint32_t carry = 0;        // bytes of an unfinished line at tile[t0..t0+carry)
    // the tile's data starts at t0 < 16, kept such that tile + t0 + carry and the next source byte have the same alignment
    // modulo 16: every 16-byte load from global memory is then a 16-byte store to shared memory
    uint32_t t0 = (uint32_t)((uintptr_t)(P.bytes + sb) & 15u);
    while (pos < se || carry) {
      // ---- stage the next tile after the carry
      uint32_t room = kTile - carry;
      uint32_t take = (uint32_t)((se - pos) < room ? (se - pos) : room);
      if (take == 0 && pos >= se) break;  // only an unterminated tail is left: the reference never parses it
      {
        // global → shared; source alignment is arbitrary, so align the 16-byte loads on the source
        const uint8_t* g = P.bytes + pos;
        uint32_t head = (uint32_t)((16 - ((uintptr_t)g & 15)) & 15); if (head > take) head = take;
        uint8_t* dst = tile + t0 + carry;
        for (uint32_t i = lane; i < head; i += 32) dst[i] = g[i];
        const uint32_t body = (take - head) & ~15u;
        const uint4* g4 = (const uint4*)(g + head);
        uint4* d4 = (uint4*)(dst + head);
        for (uint32_t i = lane; i < (body >> 4); i += 32) d4[i] = __ldg(g4 + i);
        for (uint32_t i = head + body + lane; i < take; i += 32) dst[i] = g[i];
      }
      __syncwarp();
      const uint32_t filled = carry + take;
      const uint64_t tile_base = pos - carry - t0;  // stream offset of tile[0]
      pos += take;
      // ---- newline positions and walk candidates, 16 bytes per lane per step (SIMD-in-register byte compares)
      uint32_t nlines = 0; bool overflow = false;
      uint32_t ncand = 0;
      if (lane < kMaxLines / 32) s_need[lane] = 0;
      {
        const uint32_t lo = t0, hi = t0 + filled;
        for (uint32_t cb0 = 0; cb0 < hi; cb0 += 512u) {
          const uint32_t off = cb0 + ((uint32_t)lane << 4);
          uint32_t mn = 0, mq = 0, mb = 0, mu = 0;
          if (off < hi) {
            const uint4 v = *(const uint4*)(tile + off);
            const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
              mn |= nib_ff(__vcmpeq4(w[j], 0x0a0a0a0au)) << (4 * j);
              mq |= nib_ff(__vcmpeq4(w[j], 0x22222222u)) << (4 * j);
              mb |= nib_ff(__vcmpeq4(w[j], 0x5c5c5c5cu)) << (4 * j);
              mu |= nib_ff(__vcmpeq4(w[j], 0x75757575u)) << (4 * j);
            }
            // bytes of this chunk inside [lo, hi)
            uint32_t vm = 0xffffu;
            if (off < lo) vm &= lo - off >= 16u ? 0u : (0xffffu << (lo - off));
            if (off + 16u > hi) vm &= (1u << (hi - off)) - 1u;
            mn &= vm;
            const uint32_t next_u = tile[off + 16] == 'u' ? 0x8000u : 0u;
            uint32_t cand = (mq | mb) & ((mu >> 1) | next_u) & vm;
            // `"u…`: keep only a full `"usage"`
            uint32_t cq = cand & mq;
            while (cq) {
              const int j = __ffs(cq) - 1; cq &= cq - 1;
              const uint8_t* q = tile + off + j;
              if (!(off + j + 6 < hi && q[2] == 's' && q[3] == 'a' && q[4] == 'g' && q[5] == 'e' && q[6] == '"')) cand &= ~(1u << j);
            }
            mq = cand;   // reuse: surviving candidates
          } else mq = 0;
          // newlines → lstart (warp scan of the per-lane counts)
          const uint32_t cnt = __popc(mn);
          uint32_t incl = cnt;
#pragma unroll
          for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t t = __shfl_up_sync(FULLM, incl, sft); if (lane >= sft) incl += t; }
          uint32_t k = nlines + incl - cnt;
          while (mn) { const int j = __ffs(mn) - 1; mn &= mn - 1; if (k < kMaxLines) lstart[k] = (uint16_t)(off + j); else overflow = true; k++; }
          nlines += __shfl_sync(FULLM, incl, 31);
          // candidate positions → list (resolved to lines once lstart is complete)
          const uint32_t cm = __ballot_sync(FULLM, mq != 0);
          if (cm) {
            const uint32_t c2 = __popc(mq);
            uint32_t in2 = c2;
#pragma unroll
            for (int sft = 1; sft < 32; sft <<= 1) { const uint32_t t = __shfl_up_sync(FULLM, in2, sft); if (lane >= sft) in2 += t; }
            uint32_t kk = ncand + in2 - c2;
            while (mq) { const int j = __ffs(mq) - 1; mq &= mq - 1; if (kk < kMaxCand) s_cand[kk] = (uint16_t)(off + j); kk++; }
            ncand += __shfl_sync(FULLM, in2, 31);
          }
        }
      }
      overflow = __any_sync(FULLM, overflow);
      __syncwarp();
      if (nlines == 0) {
        if (filled >= (uint32_t)kTile) { status = AIGW_DECLINED; break; }  // a single line longer than the tile
        if (pos >= se) break;
        carry = filled; continue;
      }
      if (overflow) { status = AIGW_DECLINED; break; }
      __syncwarp();
      const bool cand_overflow = ncand > (uint32_t)kMaxCand;   // too many candidates to list: walk every line of this tile
      if (!cand_overflow) {
        for (uint32_t c = lane; c < ncand; c += 32) {
          const uint32_t p = s_cand[c];
          uint32_t lo2 = 0, hi2 = nlines;   // first line whose newline lies behind p
          while (lo2 < hi2) { const uint32_t mid = (lo2 + hi2) >> 1; if (lstart[mid] > p) hi2 = mid; else lo2 = mid + 1; }
          if (lo2 < nlines) atomicOr(&s_need[lo2 >> 5], 1u << (lo2 & 31));
        }
      }
      __syncwarp();
      // ---- which lines need the typed walk?
      // A line changes the usage only if it decodes AND carries a top-level "usage" member; it changes the response model
      // only if it is the LAST decodable line with a non-empty model.  So a line is walked when it contains the bytes
      // `"usage"` (keys are matched case-sensitively, internal/json/json.go) or a `\u` escape (which could spell that key),
      // or when it is one of the last two `data: ` lines of the tile (model candidates).  If neither candidate yields a model
      // the whole tile is walked again without the filter, so the result is the reference's for every input.
      uint32_t cand1 = 0xffffffffu, cand2 = 0xffffffffu;   // the tile's last and second-to-last data line
      for (uint32_t l0 = 0; l0 < nlines; l0 += 32) {
        const uint32_t li = l0 + lane;
        bool isd = false;
        if (li < nlines) { const int b = li == 0 ? (int)t0 : lstart[li - 1] + 1; const int e = lstart[li]; const uint8_t* q = tile + b; isd = e - b >= 6 && q[0] == 'd' && q[1] == 'a' && q[2] == 't' && q[3] == 'a' && q[4] == ':' && q[5] == ' '; }
        const uint32_t m = __ballot_sync(FULLM, isd);
        if (m) {   // groups ascend, so this group's top two data lines supersede the earlier candidates
          const uint32_t hi = 31u - __clz(m), m2 = m & ~(1u << hi);
          cand2 = m2 ? l0 + (31u - __clz(m2)) : cand1;
          cand1 = l0 + hi;
        }
      }
      for (int pass = 0; pass < 2; pass++) {
        const bool walk_all = pass == 1;
        uint32_t model_found = 0;
        for (uint32_t l0 = 0; l0 < nlines; l0 += 32) {
          const uint32_t li = l0 + lane;
          if (li < nlines) {
            const int b = li == 0 ? (int)t0 : lstart[li - 1] + 1;
            const int e = lstart[li];
            const uint8_t* q = tile + b; const int n = e - b;
            if (n >= 6 && q[0] == 'd' && q[1] == 'a' && q[2] == 't' && q[3] == 'a' && q[4] == ':' && q[5] == ' ') {
              const bool need = walk_all || cand_overflow || li == cand1 || li == cand2 || ((s_need[li >> 5] >> (li & 31)) & 1u);
              if (need) {
                Capture cp; cp.int_set = 0; cp.obj_seen = 0; cp.span_set = 0; cp.span_esc = 0; cp.weird = 0; cp.big = 0;
#pragma unroll
                for (int k = 0; k < 8; k++) cp.ints[k] = 0;
                const bool ok = walk(q + 6, n - 6, sch->nodes, sch->fields, sch->keys, N_ROOT, cp);
                if (cp.weird || (cp.span_esc & 1u)) status = AIGW_DECLINED;
                if (ok) {
                  const uint32_t seq = line_no + li + 1;
                  if ((cp.span_set & 1u) && cp.span_len[0] > 0) { if (seq >= seq_m) { seq_m = seq; m_off = tile_base + (uint64_t)b + 6 + cp.span_off[0]; m_len = cp.span_len[0]; } if (li == cand1 || li == cand2) model_found = 1; }
                  if (cp.obj_seen & (1u << C_OBJ_USAGE)) {
                    if (seq >= seq_u) { seq_u = seq; v_in = cp.ints[C_PROMPT]; v_out = cp.ints[C_COMPLETION]; v_tot = cp.ints[C_TOTAL]; }
                    if ((cp.obj_seen & (1u << C_OBJ_PTD)) && seq >= seq_p) { seq_p = seq; v_cached = cp.ints[C_CACHED]; v_cc = cp.ints[C_CACHE_CREATION]; }
                    if ((cp.obj_seen & (1u << C_OBJ_CTD)) && seq >= seq_c) { seq_c = seq; v_reason = cp.ints[C_REASONING]; }
                  }
                }
              }
            }
          }
        }
        // a candidate that decoded with a non-empty model is the tile's last such line (only the other, later candidate could
        // follow it, and it was walked too); otherwise walk every line of the tile
        if (walk_all || cand1 == 0xffffffffu || __any_sync(FULLM, model_found)) break;
      }
      __syncwarp();
      line_no += nlines;
      // ---- carry the unterminated tail to the front of the tile, at the offset that keeps the staging aligned
      const uint32_t last = (uint32_t)lstart[nlines - 1] + 1;
      const uint32_t rem = t0 + filled - last;
      const uint32_t nt0 = (uint32_t)(((uintptr_t)(P.bytes + pos) - rem) & 15u);
      if (rem && nt0 != last) {
        const uint32_t nchunk = (rem + 31u) >> 5;
        for (uint32_t k = 0; k < nchunk; k++) {
          const uint32_t ck = nt0 <= last ? k : nchunk - 1u - k;   // ascending when moving down, descending when moving up
          const uint32_t i = (ck << 5) + lane;
          uint8_t c = 0; if (i < rem) c = tile[last + i];
          __syncwarp();
          if (i < rem) tile[nt0 + i] = c;
          __syncwarp();
        }
      }
      t0 = nt0;
      carry = rem;
      if (pos >= se) break;
    }
    // ---- latest-wins merge across lanes
    status = __reduce_or_sync(FULLM, status);
    aigw_sse_result r; memset(&r, 0, sizeof r);
    auto pick = [&](uint32_t seq) -> int { const uint32_t mx = __reduce_max_sync(FULLM, seq); if (mx == 0) return -1; const uint32_t who = __ballot_sync(FULLM, seq == mx); return __ffs(who) - 1; };
    int w;
    w = pick(seq_u); if (w >= 0) { r.usage.input = __shfl_sync(FULLM, v_in, w); r.usage.output = __shfl_sync(FULLM, v_out, w); r.usage.total = __shfl_sync(FULLM, v_tot, w); r.usage.mask |= 1u | 2u | 4u; }
    w = pick(seq_p); if (w >= 0) { r.usage.cached = __shfl_sync(FULLM, v_cached, w); r.usage.cache_creation = __shfl_sync(FULLM, v_cc, w); r.usage.mask |= 8u | 16u; }
    w = pick(seq_c); if (w >= 0) { r.usage.reasoning = __shfl_sync(FULLM, v_reason, w); r.usage.mask |= 32u; }
    w = pick(seq_m); if (w >= 0) { r.model_off = __shfl_sync(FULLM, m_off, w); r.model_len = __shfl_sync(FULLM, m_len, w); }
    r.status = status;
    if (lane == 0) P.results[s] = r;
  }
}

// R1: non-stream ChatCompletionResponse usage — the schema table (enum RN, kRespFields, build_resp_schema) lives in sse_schema.cuh
__device__ RespSchemaBlob g_resp_schema;

// openai.EmbeddingResponse (internal/apischema/openai/openai.go:1683-1731,1772-1778): R_ROOT fields differ, so a second blob
static const FieldDef kEmbFields[] = {
  {R_ROOT, "object", R_STR}, {R_ROOT, "data", R_EM_DATA}, {R_ROOT, "model", R_MODEL}, {R_ROOT, "usage", R_EM_USAGE},
  {R_EM_ITEM, "object", R_STR}, {R_EM_ITEM, "embedding", R_EM_VEC}, {R_EM_ITEM, "index", R_INT},
  {R_EM_USAGE, "prompt_tokens", R_PROMPT}, {R_EM_USAGE, "total_tokens", R_TOTAL},
};
__device__ RespSchemaBlob g_emb_schema;
static RespSchemaBlob build_emb_schema() {
  RespSchemaBlob b; memset(&b, 0, sizeof b);
  auto set = [&](int n, uint8_t kind, uint8_t cap = NOCAP, uint8_t elem = 0) { b.nodes[n].kind = kind; b.nodes[n].cap = cap; b.nodes[n].elem = elem; };
  set(R_ANY, K_ANY); set(R_STR, K_STR); set(R_INT, K_INT); set(R_FLOAT, K_FLOAT);
  set(R_ROOT, K_OBJ); set(R_EM_DATA, K_ARR, NOCAP, R_EM_ITEM); set(R_EM_ITEM, K_OBJ);
  set(R_EM_VEC, K_STROBJ, NOCAP, R_EM_FLOATS);   // EmbeddingUnion: a string, or (the alternative node) an array of numbers
  set(R_EM_FLOATS, K_ARR, NOCAP, R_FLOAT);
  set(R_EM_USAGE, K_OBJ, C_OBJ_USAGE); set(R_MODEL, K_STR, C_SPAN_MODEL); set(R_PROMPT, K_INT, C_PROMPT); set(R_TOTAL, K_INT, C_TOTAL);
  int ko = 0;
  for (int f = 0; f < (int)(sizeof(kEmbFields) / sizeof(kEmbFields[0])); f++) {
    const FieldDef& d = kEmbFields[f];
    Node& o = b.nodes[d.owner];
    if (o.nf == 0) o.f0 = (uint8_t)f;
    o.nf++;
    int kl = (int)strlen(d.key);
    b.fields[f].koff = (uint16_t)ko; b.fields[f].klen = (uint8_t)kl; b.fields[f].node = d.node;
    memcpy(b.keys + ko, d.key, kl); ko += kl;
  }
  return b;
}

// one thread per response body; `embeddings`: openai.EmbeddingResponse instead of openai.ChatCompletionResponse
__global__ void __launch_bounds__(128) response_usage_kernel(const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results, int embeddings) {
  __shared__ RespSchemaBlob sch;
  for (uint32_t i = threadIdx.x; i < sizeof(RespSchemaBlob) / 4; i += blockDim.x) ((uint32_t*)&sch)[i] = ((const uint32_t*)(embeddings ? &g_emb_schema : &g_resp_schema))[i];
  __syncthreads();
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n) return;
  const uint8_t* p = bodies + offsets[d];
  Capture cp; cp.int_set = 0; cp.obj_seen = 0; cp.span_set = 0; cp.span_esc = 0; cp.weird = 0; cp.big = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) cp.ints[k] = 0;
  const bool ok = walk(p, (int)lens[d], sch.nodes, sch.fields, sch.keys, R_ROOT, cp, /*allow_trailing=*/true);
  aigw_sse_result r; memset(&r, 0, sizeof r);
  if (cp.weird || (cp.span_esc & 1u)) r.status = AIGW_DECLINED;
  else if (!ok) r.status = AIGW_INTERNAL;  // "failed to unmarshal body": the reference fails the request
  else {
    // resp.Usage is a value: the three counters are always set; details only when their object was present
    r.usage.input = cp.ints[C_PROMPT]; r.usage.output = cp.ints[C_COMPLETION]; r.usage.total = cp.ints[C_TOTAL]; r.usage.mask = embeddings ? (1u | 4u) : (1u | 2u | 4u);
    if (cp.obj_seen & (1u << C_OBJ_PTD)) { r.usage.cached = cp.ints[C_CACHED]; r.usage.cache_creation = cp.ints[C_CACHE_CREATION]; r.usage.mask |= 8u | 16u; }
    if (cp.obj_seen & (1u << C_OBJ_CTD)) { r.usage.reasoning = cp.ints[C_REASONING]; r.usage.mask |= 32u; }
    if ((cp.span_set & 1u) && cp.span_len[0] > 0) { r.model_off = offsets[d] + cp.span_off[0]; r.model_len = cp.span_len[0]; }
  }
  results[d] = r;
}

// Buffered /v1/completions responses (openai_completions.go:98-150): json.Unmarshal of the whole body (no trailing bytes) into
// openai.CompletionResponse; responseModel = resp.Model; every counter is set only when it is >= 0 — a negative or >= 2^31
// counter is outside the integer captures' range and DECLINES.  The schema is read in place from device memory.
__device__ SchemaBlob g_cmpl_resp_schema;
__global__ void __launch_bounds__(128) completions_response_kernel(const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x;
  if (d >= n) return;
  const uint8_t* p = bodies + offsets[d];
  Capture cp; cp.int_set = 0; cp.obj_seen = 0; cp.span_set = 0; cp.span_esc = 0; cp.weird = 0; cp.big = 0;
#pragma unroll
  for (int k = 0; k < 8; k++) cp.ints[k] = 0;
  const bool ok = walk(p, (int)lens[d], g_cmpl_resp_schema.nodes, g_cmpl_resp_schema.fields, g_cmpl_resp_schema.keys, N_ROOT, cp, /*allow_trailing=*/false);
  aigw_sse_result r; memset(&r, 0, sizeof r);
  if (cp.weird || (cp.span_esc & 1u)) r.status = AIGW_DECLINED;
  else if (!ok) r.status = AIGW_INTERNAL;  // "failed to unmarshal body"
  else {
    if (cp.obj_seen & (1u << C_OBJ_USAGE)) {
      if (cp.big) r.status = AIGW_DECLINED;
      else {
        r.usage.input = cp.ints[C_PROMPT]; r.usage.output = cp.ints[C_COMPLETION]; r.usage.total = cp.ints[C_TOTAL]; r.usage.mask = 1u | 2u | 4u;
        if (cp.obj_seen & (1u << C_OBJ_PTD)) { r.usage.cached = cp.ints[C_CACHED]; r.usage.cache_creation = cp.ints[C_CACHE_CREATION]; r.usage.mask |= 8u | 16u; }
        if (cp.obj_seen & (1u << C_OBJ_CTD)) { r.usage.reasoning = cp.ints[C_REASONING]; r.usage.mask |= 32u; }
      }
    }
    if ((cp.span_set & 1u) && cp.span_len[0] > 0) { r.model_off = offsets[d] + cp.span_off[0]; r.model_len = cp.span_len[0]; }
  }
  results[d] = r;
}

// C2: evalCost's direct selectors over a table of usages (internal/extproc/processor_impl.go:707-756)
__global__ void usage_costs_kernel(const aigw_sse_result* results, uint32_t n, const int32_t* cost_types, uint32_t n_costs, unsigned long long* out) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * n_costs) return;
  const aigw_usage& u = results[i / n_costs].usage;
  unsigned long long v = 0;
  switch (cost_types[i % n_costs]) { case 0: v = u.input; break; case 1: v = u.cached; break; case 2: v = u.cache_creation; break; case 3: v = u.output; break; case 4: v = u.total; break; case 5: v = u.reasoning; break; default: v = 0; }
  out[i] = v;
}

cudaError_t launch_response_usage(const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results, cudaStream_t st, int embeddings) {
  static DeviceOnce once;
  {
    const cudaError_t e0 = device_once(once, nullptr, [&](int*) {
      RespSchemaBlob b = build_resp_schema(); cudaError_t e = cudaMemcpyToSymbol(g_resp_schema, &b, sizeof b); if (e != cudaSuccess) return e;
      RespSchemaBlob b2 = build_emb_schema(); e = cudaMemcpyToSymbol(g_emb_schema, &b2, sizeof b2); if (e != cudaSuccess) return e;
      SchemaBlob b3 = build_completion_schema(); return cudaMemcpyToSymbol(g_cmpl_resp_schema, &b3, sizeof b3);
    });
    if (e0 != cudaSuccess) return e0;
  }
  if (n == 0) return cudaSuccess;
  if (embeddings == 2) { completions_response_kernel<<<(n + 127) / 128, 128, 0, st>>>(bodies, offsets, lens, n, results); return cudaGetLastError(); }
  response_usage_kernel<<<(n + 127) / 128, 128, 0, st>>>(bodies, offsets, lens, n, results, embeddings);
  return cudaGetLastError();
}
cudaError_t launch_usage_costs(const aigw_sse_result* results, uint32_t n, const int32_t* cost_types, uint32_t n_costs, unsigned long long* out, cudaStream_t st) {
  if (n == 0 || n_costs == 0) return cudaSuccess;
  const uint32_t tot = n * n_costs;
  usage_costs_kernel<<<(tot + 255) / 256, 256, 0, st>>>(results, n, cost_types, n_costs, out);
  return cudaGetLastError();
}

cudaError_t launch_sse_usage(const SseParams& P, int sm_count, cudaStream_t st) {
  static DeviceOnce once;
  const size_t smem = ((sizeof(SchemaBlob) + 15) & ~15u) + (size_t)kWarps * kWarpBytes;
  int* v = nullptr;
  {
    const cudaError_t e0 = device_once(once, &v, [&](int* val) {
      SchemaBlob b = build_schema();
      cudaError_t e = cudaMemcpyToSymbol(g_schema, &b, sizeof b);
      if (e != cudaSuccess) return e;
      if ((e = cudaFuncSetAttribute(sse_usage_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)) != cudaSuccess) return e;
      if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&val[0], sse_usage_kernel, kWarps * 32, smem)) != cudaSuccess) return e;
      if (val[0] < 1) val[0] = 1;
      return cudaSuccess;
    });
    if (e0 != cudaSuccess) return e0;
  }
  const int bps = v[0];
  long long want = ((long long)P.n_streams + kWarps - 1) / kWarps;
  long long grid = (long long)sm_count * bps;
  if (want < grid) grid = want;
  if (grid < 1) grid = 1;
  sse_usage_kernel<<<(unsigned)grid, kWarps * 32, smem, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
