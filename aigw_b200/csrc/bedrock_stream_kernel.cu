// See bedrock_stream_kernel.cuh.  sm_90a only.
#include <cstring>

#include "bedrock_common.cuh"
#include "device_once.cuh"

namespace aigw {

namespace {
__device__ BedrockSchema g_bedrock_schema;

constexpr int kTile = 8192;        // bytes of a stream staged per warp; also the largest frame handled
constexpr int kMaxFrames = 512;    // kTile / 16
constexpr int kWarps = 4;
constexpr int kOutTile = 12288;    // emit kernel staging per warp
constexpr int kEmitWarps = 4;

// ------------------------------------------------------------------ frames kernel
__global__ void __launch_bounds__(kWarps * 32) bedrock_frames_kernel(const __grid_constant__ BedrockStreamParams P) {
  extern __shared__ __align__(16) uint8_t smem[];
  BedrockSchema* sch = (BedrockSchema*)smem;
  uint32_t* crc_tab = (uint32_t*)(smem + ((sizeof(BedrockSchema) + 15) & ~15u));
  for (uint32_t i = threadIdx.x; i < sizeof(BedrockSchema) / 4; i += blockDim.x) ((uint32_t*)sch)[i] = ((const uint32_t*)&g_bedrock_schema)[i];
  for (uint32_t i = threadIdx.x; i < 256; i += blockDim.x) { uint32_t c = i; for (int k = 0; k < 8; k++) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1; crc_tab[i] = c; }
  __syncthreads();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t FULLM = 0xffffffffu;
  uint8_t* tile = (uint8_t*)(crc_tab + 256) + (size_t)warp * (kTile + 32 + kMaxFrames * 2);
  uint16_t* fstart = (uint16_t*)(tile + kTile + 32);

  for (;;) {
    uint32_t s = 0;
    if (lane == 0) s = atomicAdd(P.next, 1u);
    s = __shfl_sync(FULLM, s, 0);
    if (s >= P.n_streams) break;
    const uint64_t sb = P.stream_off[s], se = P.stream_off[s + 1];
    BedrockRec* recs = P.recs + ((sb - P.off_base) >> 5) + 2ull * s;
    const uint32_t rec_cap = (uint32_t)((se - sb) >> 5) + 2u;
    uint32_t nrec = 0, out_total = 0;
    uint32_t status = 0, reason = 0;
    // stream state threaded through the events (openai_awsbedrock.go:43-47)
    uint32_t role_off = 0, role_len = 0, tool_index = 0; bool active_tool = false;
    aigw_usage usage; memset(&usage, 0, sizeof usage);
    uint64_t pos = sb; uint32_t carry = 0; bool blocked = false;
    // data lives at tile[t0 .. t0+filled), t0 < 16 chosen so that shared and global addresses agree modulo 16 (aligned 16-byte staging)
    uint32_t t0 = (uint32_t)((uintptr_t)(P.bytes + sb) & 15u);
    uint64_t consumed = 0;
    while (!blocked && !status && (pos < se)) {
      const uint32_t room = kTile - carry;
      const uint32_t take = (uint32_t)((se - pos) < room ? (se - pos) : room);
      {
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
      const uint32_t tile_rel = (uint32_t)(pos - carry - sb) - t0;  // stream-relative offset of tile[0] (wraps consistently)
      pos += take;
      // ---- lane 0: frame chain (prelude length + prelude CRC), eventstream decoder order of checks
      uint32_t nf = 0, end = 0, chain = 0;  // chain: 0 ran out of bytes, 1 blocked by a bad prelude, 2 frame larger than the tile
      if (lane == 0) {
        uint32_t i = t0;
        const uint32_t hi = t0 + filled;
        while (i + 12 <= hi) {
          const uint8_t* f = tile + i;
          const uint32_t total = be32(f), hlen = be32(f + 4);
          uint32_t c = 0xffffffffu;
#pragma unroll
          for (int k = 0; k < 8; k++) c = crc_tab[(c ^ f[k]) & 0xffu] ^ (c >> 8);
          if (~c != be32(f + 8)) { chain = 1; break; }
          if (hlen > 128u * 1024u || total < 16u || hlen > total - 16u || total - hlen - 16u > 16u * 1024u * 1024u) { chain = 1; break; }
          if (total > (uint32_t)kTile) { chain = 2; break; }
          if (i + total > hi) break;
          fstart[nf++] = (uint16_t)i; i += total;
        }
        end = i;
      }
      nf = __shfl_sync(FULLM, nf, 0); end = __shfl_sync(FULLM, end, 0); chain = __shfl_sync(FULLM, chain, 0);
      __syncwarp();
      // ---- one lane per frame
      for (uint32_t f0 = 0; f0 < nf && !blocked && !status; f0 += 32) {
        const uint32_t fi = f0 + lane;
        const bool have = fi < nf;
        bool bad = false;          // decoder error on this frame: the reference never gets past it
        uint32_t kind = KD_NONE, flags = 0, decl = 0;
        BedrockRec rec; memset(&rec, 0, sizeof rec);
        bool has_usage = false; uint32_t u_in = 0, u_out = 0, u_read = 0, u_write = 0;
        uint32_t my_role_off = 0, my_role_len = 0;
        if (have) {
          const uint32_t fo = fstart[fi];
          const uint8_t* f = tile + fo;
          const uint32_t total = be32(f), hlen = be32(f + 4);
          uint32_t c = 0xffffffffu;
          for (uint32_t k = 0; k < total - 4u; k++) c = crc_tab[(c ^ f[k]) & 0xffu] ^ (c >> 8);
          if (~c != be32(f + total - 4)) bad = true;
          // headers: [name_len u8][name][type u8][value]; :event-type is a type-7 string
          const uint8_t* et = nullptr; uint32_t etl = 0;
          if (!bad) {
            uint32_t h = 12; const uint32_t hend = 12 + hlen;
            while (h < hend) {
              const uint32_t nl = f[h]; h++;
              if (h + nl + 1 > hend) { bad = true; break; }
              const uint8_t* name = f + h; h += nl;
              const uint32_t type = f[h]; h++;
              int vs;
              switch (type) { case 0: case 1: vs = 0; break; case 2: vs = 1; break; case 3: vs = 2; break; case 4: vs = 4; break; case 5: case 8: vs = 8; break; case 9: vs = 16; break; case 6: case 7: vs = -1; break; default: vs = -2; }
              if (vs == -2) { bad = true; break; }
              if (vs == -1) { if (h + 2 > hend) { bad = true; break; } vs = (f[h] << 8) | f[h + 1]; h += 2; }
              if (h + (uint32_t)vs > hend) { bad = true; break; }
              if (type == 7 && same(name, nl, ":event-type", 11)) { et = f + h; etl = (uint32_t)vs; }
              h += (uint32_t)vs;
            }
          }
          if (!bad) {
            const uint8_t* pl = f + 12 + hlen; const int pn = (int)(total - hlen - 16);
            const uint32_t pl_rel = tile_rel + fo + 12 + hlen;   // stream-relative offset of the payload
            BCap cp; cp.int_set = 0; cp.obj_seen = 0; cp.span_set = 0; cp.span_esc = 0; cp.weird = 0; cp.big = 0;
#pragma unroll
            for (int k = 0; k < 8; k++) cp.ints[k] = 0;
            bool ok;
            if (pn == 4 && pl[0] == 'n' && pl[1] == 'u' && pl[2] == 'l' && pl[3] == 'l') ok = true;  // json null leaves the zero event
            else ok = walk(pl, pn, sch->nodes, sch->fields, sch->keys, B_ROOT, cp);
            if (cp.weird) decl = 1;
            if (ok && !decl) {
              auto has = [&](int sp) { return (cp.span_set >> sp) & 1u; };
              auto span_ok = [&](int sp) { return !has(sp) || canonical(pl + cp.span_off[sp], cp.span_len[sp]); };
              if (has(S_EVT)) { et = pl + cp.span_off[S_EVT]; etl = cp.span_len[S_EVT]; if ((cp.span_esc >> S_EVT) & 1u) decl = 1; }
              if (same(et, etl, "metadata", 8)) {
                if (cp.obj_seen & (1u << O_USAGE)) {
                  kind = KD_META; has_usage = true;
                  const bool hr = (cp.int_set >> I_READ) & 1u, hw = (cp.int_set >> I_WRITE) & 1u;
                  const unsigned long long tin = (unsigned long long)cp.ints[I_IN] + (hr ? cp.ints[I_READ] : 0u) + (hw ? cp.ints[I_WRITE] : 0u);
                  if (cp.big || tin + cp.ints[I_OUT] >= 0x80000000ull) decl = 1;
                  u_in = (uint32_t)tin; u_out = cp.ints[I_OUT]; u_read = cp.ints[I_READ]; u_write = cp.ints[I_WRITE];
                  rec.a[0] = u_in; rec.a[1] = u_out; rec.a[2] = u_read; rec.a[3] = u_write;
                  if (hr) flags |= F_HAS_READ; if (hw) flags |= F_HAS_WRITE;
                  if ((cp.obj_seen & (1u << O_TIER)) && has(S_TIER) && cp.span_len[S_TIER]) { if (!span_ok(S_TIER)) decl = 1; rec.a[4] = pl_rel + cp.span_off[S_TIER]; rec.a[5] = cp.span_len[S_TIER]; }
                }
              } else if (same(et, etl, "messageStart", 12)) {
                if (has(S_ROLE)) { kind = KD_MSGSTART; if (!span_ok(S_ROLE)) decl = 1; my_role_off = pl_rel + cp.span_off[S_ROLE]; my_role_len = cp.span_len[S_ROLE]; if (my_role_len > 64u) decl = 1; }
              } else if (same(et, etl, "contentBlockDelta", 17)) {
                if (cp.obj_seen & (1u << O_DELTA)) {
                  if (has(S_TEXT)) { kind = KD_TEXT; if (!span_ok(S_TEXT)) decl = 1; rec.a[0] = pl_rel + cp.span_off[S_TEXT]; rec.a[1] = cp.span_len[S_TEXT]; }
                  else if (cp.obj_seen & (1u << O_DTOOL)) { kind = KD_TOOLDELTA; if (!span_ok(S_TOOLIN)) decl = 1; if (has(S_TOOLIN)) { rec.a[0] = pl_rel + cp.span_off[S_TOOLIN]; rec.a[1] = cp.span_len[S_TOOLIN]; } }
                  else if (cp.obj_seen & (1u << O_DREASON)) {
                    kind = KD_REASON;
                    if (!span_ok(S_RTEXT) || !span_ok(S_RSIG)) decl = 1;
                    if (has(S_RTEXT)) { rec.a[0] = pl_rel + cp.span_off[S_RTEXT]; rec.a[1] = cp.span_len[S_RTEXT]; }
                    if (has(S_RSIG)) { rec.a[2] = pl_rel + cp.span_off[S_RSIG]; rec.a[3] = cp.span_len[S_RSIG]; }
                    if (has(S_REDACT) && cp.span_len[S_REDACT]) decl = 1;   // re-encoded []byte: left to the stock path
                  } else kind = KD_EMPTY;
                }
              } else if (same(et, etl, "contentBlockStart", 17)) {
                if (cp.obj_seen & (1u << O_START)) {
                  if (cp.obj_seen & (1u << O_STOOL)) {
                    kind = KD_TOOLSTART;
                    if (!span_ok(S_NAME) || !span_ok(S_TUID)) decl = 1;
                    if (has(S_NAME)) { rec.a[0] = pl_rel + cp.span_off[S_NAME]; rec.a[1] = cp.span_len[S_NAME]; }
                    if (has(S_TUID)) { rec.a[2] = pl_rel + cp.span_off[S_TUID]; rec.a[3] = cp.span_len[S_TUID]; }
                  } else kind = KD_EMPTY;
                }
              } else if (same(et, etl, "messageStop", 11)) {
                if (has(S_STOP)) {
                  kind = KD_STOP;
                  if ((cp.span_esc >> S_STOP) & 1u) decl = 1;
                  const uint8_t* q = pl + cp.span_off[S_STOP]; const uint32_t ql = cp.span_len[S_STOP];
                  if (same(q, ql, "max_tokens", 10)) flags |= 1u; else if (same(q, ql, "content_filtered", 16)) flags |= 2u; else if (same(q, ql, "tool_use", 8)) flags |= 3u;
                }
              } else if (same(et, etl, "contentBlockStop", 16)) kind = KD_BLOCKSTOP;
            }
          }
        }
        // ---- frames behind the first decoder error do not exist for the reference
        const uint32_t badm = __ballot_sync(FULLM, bad);
        const uint32_t livem = badm ? ((1u << (__ffs(badm) - 1)) - 1u) : FULLM;
        const bool live = have && ((livem >> lane) & 1u);
        if (!live) { kind = KD_NONE; has_usage = false; decl = 0; }
        if (badm) { blocked = true; consumed = (uint64_t)(uint32_t)(tile_rel + fstart[f0 + __ffs(badm) - 1]); }
        if (__any_sync(FULLM, decl != 0)) { status = AIGW_DECLINED; reason = AIGW_R_UNSUPPORTED_FIELD; break; }
        // ---- stream state in event order: role of the latest messageStart, tool-call index
        const uint32_t startm = __ballot_sync(FULLM, kind == KD_MSGSTART);
        const uint32_t toolm = __ballot_sync(FULLM, kind == KD_TOOLSTART);
        const uint32_t stopm = __ballot_sync(FULLM, kind == KD_BLOCKSTOP);
        {
          const uint32_t upto = startm & ((2u << lane) - 1u);          // messageStart frames at or before me
          const int src = upto ? 31 - __clz(upto) : 0;
          const uint32_t ro = __shfl_sync(FULLM, my_role_off, src), rl = __shfl_sync(FULLM, my_role_len, src);
          rec.role_off = upto ? ro : role_off; rec.role_len = upto ? rl : role_len;
          if (startm) { const int last = 31 - __clz(startm); role_off = __shfl_sync(FULLM, my_role_off, last); role_len = __shfl_sync(FULLM, my_role_len, last); }
        }
        {
          uint32_t ti = tool_index; bool act = active_tool; uint32_t mine = ti;
          for (int j = 0; j < 32; j++) {
            if (j == lane) mine = ti;
            if ((toolm >> j) & 1u) act = true;
            if (((stopm >> j) & 1u) && act) { ti++; act = false; }
          }
          rec.tool_index = mine; tool_index = ti; active_tool = act;
        }
        // ---- usage returned by the call that carries this frame, merged latest-set-wins (metrics.go:258-283)
        {
          const uint32_t um = __ballot_sync(FULLM, has_usage);
          if (um) { const int l = 31 - __clz(um); usage.input = __shfl_sync(FULLM, u_in, l); usage.output = __shfl_sync(FULLM, u_out, l); usage.total = usage.input + usage.output; usage.mask |= 7u; }
          const uint32_t rm = __ballot_sync(FULLM, has_usage && (flags & F_HAS_READ));
          if (rm) { usage.cached = __shfl_sync(FULLM, u_read, 31 - __clz(rm)); usage.mask |= 8u; }
          const uint32_t wm = __ballot_sync(FULLM, has_usage && (flags & F_HAS_WRITE));
          if (wm) { usage.cache_creation = __shfl_sync(FULLM, u_write, 31 - __clz(wm)); usage.mask |= 16u; }
        }
        // ---- size the chunk, hand out record slots
        const bool emits = kind != KD_NONE && kind != KD_BLOCKSTOP;
        rec.kf = kind | (flags << 8);
        if (emits) rec.out_len = emit_chunk<false>(rec, P, nullptr, nullptr);
        const uint32_t em = __ballot_sync(FULLM, emits);
        const uint32_t slot = nrec + __popc(em & ((1u << lane) - 1u));
        if (nrec + __popc(em) > rec_cap) { status = AIGW_DECLINED; reason = AIGW_R_OPS; break; }
        if (emits) recs[slot] = rec;
        nrec += __popc(em);
        uint32_t ol = emits ? rec.out_len : 0u;
#pragma unroll
        for (int d = 16; d; d >>= 1) ol += __shfl_xor_sync(FULLM, ol, d);
        out_total += ol;
      }
      if (blocked || status) break;
      if (chain == 1) { blocked = true; consumed = (uint64_t)(uint32_t)(tile_rel + end); break; }
      if (chain == 2) { status = AIGW_DECLINED; reason = AIGW_R_TOO_LARGE; break; }
      // ---- carry the incomplete frame to the front of the tile, at the offset that keeps the staging aligned
      const uint32_t rem = t0 + filled - end;
      consumed = (uint64_t)(uint32_t)(tile_rel + end);
      if (end != t0) {
        const uint32_t nt0 = (uint32_t)(((uintptr_t)(P.bytes + pos) - rem) & 15u);
        if (rem && nt0 != end) {
          const uint32_t nchunk = (rem + 31u) >> 5;
          for (uint32_t k = 0; k < nchunk; k++) {
            const uint32_t ck = nt0 <= end ? k : nchunk - 1u - k;
            const uint32_t i = (ck << 5) + lane;
            uint8_t c = 0; if (i < rem) c = tile[end + i];
            __syncwarp();
            if (i < rem) tile[nt0 + i] = c;
            __syncwarp();
          }
        }
        t0 = nt0;
      }
      carry = rem;
    }
    // ---- stream result + output range
    if (lane == 0) {
      aigw_stream_result r; memset(&r, 0, sizeof r);
      r.status = status; r.reason = reason; r.consumed = consumed; r.n_chunks = nrec;
      if (!status) {
        const uint32_t total = out_total + (uint32_t)(sizeof(L_DONE) - 1);
        const unsigned long long o = atomicAdd(P.out_used, (unsigned long long)((total + 15u) & ~15u));
        if (o + total > P.out_capacity) { r.status = AIGW_DECLINED; r.reason = AIGW_R_ARENA_FULL; nrec = 0; }
        else { r.out_off = o + P.out_bias; r.out_len = total; r.usage = usage; }
      }
      P.results[s] = r;
      P.rec_count[s] = r.status ? 0xffffffffu : nrec;
      P.out_pos[s] = r.out_off - P.out_bias;
    }
  }
}

// ------------------------------------------------------------------ emit kernel
__global__ void __launch_bounds__(kEmitWarps * 32) bedrock_emit_kernel(const __grid_constant__ BedrockStreamParams P) {
  extern __shared__ __align__(16) uint8_t smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const uint32_t FULLM = 0xffffffffu;
  uint8_t* tile = smem + (size_t)warp * (kOutTile + 32);
  for (;;) {
    uint32_t s = 0;
    if (lane == 0) s = atomicAdd(P.next + 1, 1u);
    s = __shfl_sync(FULLM, s, 0);
    if (s >= P.n_streams) break;
    const uint32_t nrec = P.rec_count[s];
    if (nrec == 0xffffffffu) continue;
    const uint64_t sb = P.stream_off[s];
    const BedrockRec* recs = P.recs + ((sb - P.off_base) >> 5) + 2ull * s;
    const uint8_t* src = P.bytes + sb;
    uint8_t* g = P.out + P.out_pos[s];
    // warp flush of tile[a .. a+len) to g (a == g & 15, so 16-byte stores line up on both sides)
    auto flush = [&](uint32_t len) {
      const uint32_t a = (uint32_t)((uintptr_t)g & 15u);
      uint32_t head = (16u - a) & 15u; if (head > len) head = len;
      if (lane < (int)head) g[lane] = tile[a + lane];
      const uint32_t body = (len - head) & ~15u;
      const uint4* t4 = (const uint4*)(tile + a + head);
      uint4* g4 = (uint4*)(g + head);
      for (uint32_t i = lane; i < (body >> 4); i += 32) g4[i] = t4[i];
      for (uint32_t i = head + body + lane; i < len; i += 32) g[i] = tile[a + i];
      g += len;
    };
    uint32_t r0 = 0;
    while (r0 < nrec) {
      const uint32_t ri = r0 + lane;
      BedrockRec rec; rec.out_len = 0;
      if (ri < nrec) rec = recs[ri];
      uint32_t incl = ri < nrec ? rec.out_len : 0u;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULLM, incl, d); if (lane >= d) incl += v; }
      const uint32_t fits = __ballot_sync(FULLM, ri < nrec && incl <= (uint32_t)kOutTile);
      const uint32_t take = __popc(fits);           // ≥ 1: a chunk is bounded by its frame (≤ kTile) plus fixed text
      const uint32_t a = (uint32_t)((uintptr_t)g & 15u);
      if ((uint32_t)lane < take) emit_chunk<true>(rec, P, src, tile + a + incl - rec.out_len);
      const uint32_t len = __shfl_sync(FULLM, incl, take - 1);
      __syncwarp();
      flush(len);
      __syncwarp();
      r0 += take;
    }
    {
      const uint32_t a = (uint32_t)((uintptr_t)g & 15u);
      if (lane < (int)(sizeof(L_DONE) - 1)) tile[a + lane] = (uint8_t)L_DONE[lane];
      __syncwarp();
      flush((uint32_t)(sizeof(L_DONE) - 1));
      __syncwarp();
    }
  }
}

}  // namespace

static size_t up256(size_t v) { return (v + 255) & ~(size_t)255; }
size_t bedrock_work_bytes(uint64_t total_bytes, uint32_t n_streams) {
  return (size_t)((total_bytes >> 5) + 2ull * n_streams + 2) * sizeof(BedrockRec) + up256((size_t)n_streams * 4) + up256((size_t)n_streams * 8) + 256;
}
void bedrock_work_layout(BedrockStreamParams& P, uint8_t* work, uint32_t n_streams) {
  P.rec_count = (uint32_t*)work; work += up256((size_t)n_streams * 4);
  P.out_pos = (uint64_t*)work; work += up256((size_t)n_streams * 8);
  P.recs = (BedrockRec*)work;
}

cudaError_t launch_bedrock_stream(const BedrockStreamParams& P, int sm_count, cudaStream_t st) {
  static DeviceOnce once;
  const size_t smem_a = ((sizeof(BedrockSchema) + 15) & ~15u) + 1024 + (size_t)kWarps * (kTile + 32 + kMaxFrames * 2);
  const size_t smem_b = (size_t)kEmitWarps * (kOutTile + 32);
  int* bps = nullptr;
  {
    const cudaError_t e0 = device_once(once, &bps, [&](int* v) {
      BedrockSchema b = build_schema_bedrock();
      cudaError_t e = cudaMemcpyToSymbol(g_bedrock_schema, &b, sizeof b);
      if (e != cudaSuccess) return e;
      if ((e = cudaFuncSetAttribute(bedrock_frames_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_a)) != cudaSuccess) return e;
      if ((e = cudaFuncSetAttribute(bedrock_emit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_b)) != cudaSuccess) return e;
      if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v[0], bedrock_frames_kernel, kWarps * 32, smem_a)) != cudaSuccess) return e;
      if ((e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&v[1], bedrock_emit_kernel, kEmitWarps * 32, smem_b)) != cudaSuccess) return e;
      if (v[0] < 1) v[0] = 1;
      if (v[1] < 1) v[1] = 1;
      return cudaSuccess;
    });
    if (e0 != cudaSuccess) return e0;
  }
  const int bps_a = bps[0], bps_b = bps[1];
  if (P.n_streams == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(P.next, 0, 2 * sizeof(unsigned int), st);
  if (e != cudaSuccess) return e;
  auto grid = [&](int warps, int bps) { long long want = ((long long)P.n_streams + warps - 1) / warps, g = (long long)sm_count * bps; if (want < g) g = want; return (unsigned)(g < 1 ? 1 : g); };
  bedrock_frames_kernel<<<grid(kWarps, bps_a), kWarps * 32, smem_a, st>>>(P);
  if ((e = cudaGetLastError()) != cudaSuccess) return e;
  bedrock_emit_kernel<<<grid(kEmitWarps, bps_b), kEmitWarps * 32, smem_b, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
