// /v1/embeddings requests above the translate pass's 64 KiB ceiling (and below it): EmbeddingsEndpointSpec.ParseBody over
// openai.EmbeddingRequest and the OpenAI / Azure passthrough, the GCP Vertex AI predict request or the Amazon Titan request, with
// the semantics plan_embeddings (chat_walk_impl.cuh) gives the AIGW_SCHEMA_EMB_* schemas.  sm_90a only.
//
// emb_large_kernel: one CTA of 256 threads per request, persistent CTAs pulling requests from a counter.  The CTA that scans a
// request also plans and writes its record, so the request's token list, escape list and copy ops live in the CTA's workspace
// slice only while the CTA holds the request.
//   scan      the body streams through in 8 KB tiles (32 bytes per thread), as in rerank_scan_kernel: escapes by the odd-run
//             rule with a carry across threads and tiles, escape validation, in-string parity, token compaction.  For the Vertex
//             and Titan targets the same pass records every escape the reference's encoder spells differently (\/ \b \f \u) as
//             one entry: its position, its input width (2, 6, or 12 for a surrogate pair) and its output bytes (at most 6).
//             A lone surrogate is an entry marked bad: it declines (AIGW_R_ESCAPE) only when its string is emitted.
//   depth     bracket depth after every token by a block-wide prefix sum (depth above 48 DECLINES), the grammar of every scalar,
//             the root's first "input" array
//   input     a flat input array (no object inside) is checked in parallel: a neighbour rule for its grammar, and the element
//             types of plan_embeddings' union ([]string with nulls, ints with nulls under emb_int's rules, arrays of those); the
//             first failing element in body order wins
//   walk      thread 0 walks the root's members in body order with plan_embeddings' checks, grammar-checks and skips unknown
//             members, walks item objects (EmbeddingInputItem) serially, and plans the record as a list of copy ops: an input
//             span, a literal, a scratch span (the Titan path), or an emitted string (a span whose re-spelled escapes are taken
//             from the escape list)
//   emit      every op's output length (an emitted string: its span minus the width change of the escape entries inside it, two
//             binary searches), a block-wide prefix sum, one bump allocation, then 16-byte output chunks with every thread busy:
//             a chunk inside one span (or inside the unescaped part of a string) is one realigned 16-byte load, the others are
//             assembled byte by byte with a cursor that walks ops and escape entries.
// The failure that counts: a decline of the scan first, then a syntax error anywhere, then the first problem of the root's members
// in body order, then the input union, then the model and override checks, then the translator's 422 / 500.
#include "emb_large_kernel.cuh"

#include <string.h>

#include "classify.cuh"
#include "scan_common.cuh"
#include "scan_stream.cuh"

namespace aigw {

static constexpr int kElThreads = 256;
static constexpr uint32_t kElTile = kElThreads * 32;
static constexpr uint32_t FULL = 0xffffffffu;
// the workspace of the whole grid: at most 1 GiB
static constexpr uint64_t kElWorkspace = 1ull << 30;
enum : uint32_t { OP_SPAN = 0, OP_LIT = 1, OP_STR = 2, OP_SCR = 3 };

struct ElShared {
  uint32_t wesc[2][8], wpar[2][8], wlast[2][8], wcnt[2][8], wem[2][8];
  uint32_t wsum[2][8];
  unsigned long long wsum64[2][8];
  uint32_t doc, fail;
  uint32_t dlb, drb;                    // the root's first "input" array: its bracket and the token that closes it
  uint32_t dnest, dsyn, ifail, icount;  // input array: not flat, syntax error, first failing element (token << 8 | reason), elements
  uint32_t nops, path_len, dtotal;
  unsigned long long total;             // the record's length (path and body), saturated just above the output ceiling
  unsigned long long off;
  aigw_doc_result res;
  uint8_t lits[768];
  uint16_t lit_off[EL_COUNT], lit_len[EL_COUNT];
};

__device__ __forceinline__ uint32_t hex4(const uint8_t* p) {
  uint32_t h = 0;
  for (int k = 0; k < 4; k++) { const uint32_t c = p[k]; h = h * 16u + (c <= '9' ? c - '0' : (c | 0x20u) - 'a' + 10u); }
  return h;
}

// the escape entry of the escaped byte at p (its backslash at p - 1): x = position of the backslash | input width << 24 |
// output width << 28, y / z = output bytes 0-3 / 4-5; bad (a lone surrogate) has width 15.  Returns false when the escape is
// spelled unchanged (\" \\ \n \r \t) or is the low half of a pair (the high half's entry covers it).  `prev_esc(q)`: byte q
// is escaped (q >= p - 6).
template <class PrevEsc>
__device__ __forceinline__ bool esc_entry(const uint8_t* body, uint32_t len, uint32_t p, PrevEsc prev_esc, uint4& e) {
  const uint32_t ch = body[p];
  uint32_t cp, in = 2;
  if (ch == '/') cp = '/';
  else if (ch == 'b') cp = 8;
  else if (ch == 'f') cp = 12;
  else if (ch == 'u') {
    // a \u without four hex digits inside the body was declined by the validation: no entry, and no read past the body
    if (!(p + 4u < len && is_hex(body[p + 1]) && is_hex(body[p + 2]) && is_hex(body[p + 3]) && is_hex(body[p + 4]))) return false;
    cp = hex4(body + p + 1); in = 6;
    if (cp >= 0xD800u && cp < 0xDC00u) {
      uint32_t lo = 0;
      const bool pair = p + 10u < len && body[p + 5] == '\\' && body[p + 6] == 'u' && is_hex(body[p + 7]) && is_hex(body[p + 8]) &&
                        is_hex(body[p + 9]) && is_hex(body[p + 10]) && (lo = hex4(body + p + 7)) >= 0xDC00u && lo < 0xE000u;
      if (!pair) { e = make_uint4((p - 1u) | (6u << 24) | (15u << 28), 0, 0, 0); return true; }
      cp = 0x10000u + ((cp - 0xD800u) << 10) + (lo - 0xDC00u); in = 12;
    } else if (cp >= 0xDC00u && cp < 0xE000u) {
      if (p >= 7u && body[p - 7] == '\\' && body[p - 6] == 'u' && prev_esc(p - 6u)) {
        const uint32_t hi = hex4(body + p - 5);
        if (hi >= 0xD800u && hi < 0xDC00u) return false;
      }
      e = make_uint4((p - 1u) | (6u << 24) | (15u << 28), 0, 0, 0);
      return true;
    }
  } else return false;
  uint32_t o[6] = {0, 0, 0, 0, 0, 0}, w;
  if (cp == '"' || cp == '\\') { o[0] = '\\'; o[1] = cp; w = 2; }
  else if (cp == 10u || cp == 13u || cp == 9u) { o[0] = '\\'; o[1] = cp == 10u ? 'n' : cp == 13u ? 'r' : 't'; w = 2; }
  else if (cp < 0x20u) { const char* hx = "0123456789abcdef"; o[0] = '\\'; o[1] = 'u'; o[2] = '0'; o[3] = '0'; o[4] = (uint8_t)hx[cp >> 4]; o[5] = (uint8_t)hx[cp & 15u]; w = 6; }
  else if (cp < 0x80u) { o[0] = cp; w = 1; }
  else if (cp < 0x800u) { o[0] = 0xC0u | (cp >> 6); o[1] = 0x80u | (cp & 63u); w = 2; }
  else if (cp < 0x10000u) { o[0] = 0xE0u | (cp >> 12); o[1] = 0x80u | ((cp >> 6) & 63u); o[2] = 0x80u | (cp & 63u); w = 3; }
  else { o[0] = 0xF0u | (cp >> 18); o[1] = 0x80u | ((cp >> 12) & 63u); o[2] = 0x80u | ((cp >> 6) & 63u); o[3] = 0x80u | (cp & 63u); w = 4; }
  e = make_uint4((p - 1u) | (in << 24) | (w << 28), o[0] | (o[1] << 8) | (o[2] << 16) | (o[3] << 24), o[4] | (o[5] << 8), 0);
  return true;
}

// exclusive prefix sum of v over the CTA (values of this round), total in `tot`; wsum: 8 shared words (double-buffered by `it`)
template <class T>
__device__ __forceinline__ T block_excl(T v, T (*wsum)[8], uint32_t it, T& tot) {
  const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
  T incl = v;
#pragma unroll
  for (int s = 1; s < 32; s <<= 1) { const T x = __shfl_up_sync(FULL, incl, s); if ((int)lane >= s) incl += x; }
  if (lane == 31) wsum[it][warp] = incl;
  __syncthreads();
  T pre = 0; tot = 0;
#pragma unroll
  for (uint32_t k = 0; k < 8; k++) { const T x = wsum[it][k]; tot += x; if (k < warp) pre += x; }
  return pre + incl - v;
}

struct ElWork {
  uint32_t* tok; uint8_t* dep; uint4* esc; uint4* ops; uint8_t* scr;
};

// ---------------------------------------------------------------- the serial walk and the plan (thread 0)
struct ElPlan {
  const EmbLargeParams& P;
  const ScanToks W;
  const ElWork& w;
  uint32_t nops = 0, olen = 0;
  int err = 0;
  __device__ ElPlan(const EmbLargeParams& p, const ScanToks& t, const ElWork& wk) : P(p), W(t), w(wk) {}

  __device__ void push(uint32_t kind, uint32_t a, uint32_t y) {
    if (err) return;
    if (nops >= P.op_cap) { err = AIGW_R_OPS; return; }
    w.ops[nops++] = make_uint4((kind << 29) | a, y, 0, 0);
  }
  __device__ void span(uint32_t b, uint32_t n) { if (n) { push(OP_SPAN, b, n); olen += n; } }
  __device__ void lit(const ElShared& S, uint32_t id) { const uint32_t n = S.lit_len[id]; if (n) { push(OP_LIT, S.lit_off[id], n); olen += n; } }
  // an emitted string token j (its quotes included): the escape list gives its output length later; its token is marked emitted
  __device__ void str(uint32_t j) { push(OP_STR, W.ps(j), W.ps(j + 1)); w.dep[j] |= 0x80u; }

  __device__ uint32_t slen(uint32_t j) const { return W.ps(j + 1) - W.ps(j) - 1u; }
  __device__ bool str_is(uint32_t j, const char* k, uint32_t kl) const { const uint32_t o = W.ps(j) + 1u; return scan_key_is(W.body + o, slen(j), k, kl); }
  __device__ bool is_num(uint32_t j) const { if (W.ty(j) != T_SCALAR) return false; const uint32_t c = W.body[W.ps(j)]; return c == '-' || (c >= '0' && c <= '9'); }
  __device__ bool is_bool(uint32_t j) const { if (W.ty(j) != T_SCALAR) return false; const uint32_t c = W.body[W.ps(j)]; return c == 't' || c == 'f'; }
  __device__ bool is_null(uint32_t j) const { return W.ty(j) == T_SCALAR && W.is_null(j); }
  __device__ uint32_t after(uint32_t j) const { bool b = false; return W.skip_value(j, false, b); }
};

// emb_int (chat_walk_impl.cuh) on a scalar the depth pass found valid: 0 or the reason
__device__ __forceinline__ int emb_int_reason(const ScanToks& W, uint32_t j) {
  if (W.ty(j) != T_SCALAR) return AIGW_R_E400_TYPE;
  const uint8_t* p = W.body + W.ps(j);
  if (!(p[0] == '-' || (p[0] >= '0' && p[0] <= '9'))) return AIGW_R_E400_TYPE;
  const int k = W.scalar_kind(j);
  if (k == 3) return (p[0] == '-' && p[1] == '0') ? AIGW_R_NUMBER : 0;   // "-0" (a valid integer starting "-0" is exactly that)
  const uint32_t n = W.scalar_end(j) - W.ps(j);
  for (uint32_t i = 0; i < n; i++) if (p[i] == '.' || p[i] == 'e' || p[i] == 'E') return AIGW_R_E400_TYPE;
  return AIGW_R_NUMBER;   // more than 18 digits
}

struct ElItem { uint32_t content, task, title; };   // kNone: absent

// scan_emb_item: 0 or the reason; `empty` = EmbeddingContent.IsEmpty()
__device__ int el_item(const ElPlan& L, uint32_t e, ElItem& it, bool& empty) {
  const ScanToks& W = L.W;
  it.content = it.task = it.title = kNone; empty = true;
  if (L.is_null(e)) return 0;
  if (W.ty(e) != '{') return AIGW_R_E400_TYPE;
  uint32_t seen = 0, craw = kNone;
  if (W.ty(e + 1) != '}') for (uint32_t m = e + 1;;) {
    const uint32_t ko = W.ps(m) + 1u, kl = W.ps(m + 1) - ko;
    if (W.has_backslash(ko, ko + kl)) return AIGW_R_ESCAPE;   // keys are compared raw here (documented in the header)
    const uint8_t* kp = W.body + ko;
    const int slot = scan_key_is(kp, kl, "content", 7) ? 0 : scan_key_is(kp, kl, "task_type", 9) ? 1 : scan_key_is(kp, kl, "title", 5) ? 2 : -1;
    const uint32_t v = m + 3;
    if (slot >= 0) {
      if (seen & (1u << slot)) return AIGW_R_DUP_KEY;
      seen |= 1u << slot;
      if (slot == 0) craw = v;
      else if (!L.is_null(v)) { if (W.ty(v) != T_QOPEN) return AIGW_R_E400_TYPE; if (slot == 1) it.task = v; else it.title = v; }
    }
    const uint32_t nx = L.after(v);
    if (W.ty(nx) == '}') break;
    m = nx + 1;
  }
  if (craw != kNone) {
    if (L.is_null(craw)) empty = true;
    else if (W.ty(craw) == T_QOPEN) { it.content = craw; empty = L.slen(craw) == 0; }
    else if (W.ty(craw) == '[') {
      it.content = craw; empty = W.ty(craw + 1) == ']';
      if (!empty) for (uint32_t q = craw + 1;;) {
        if (W.ty(q) != T_QOPEN && !L.is_null(q)) return AIGW_R_E400_CONTENT;
        const uint32_t nx = L.after(q);
        if (W.ty(nx) == ']') break;
        q = nx + 1;
      }
    } else return AIGW_R_E400_CONTENT;
  }
  return 0;
}

// one gcp.Instance: {"content":C[,"task_type":T][,"title":X]} (its closing brace comes with the next one's opening)
__device__ void el_instance(ElPlan& L, const ElShared& S, uint32_t content, uint32_t task, uint32_t title, bool& first) {
  L.lit(S, first ? EL_CONTENT : EL_NEXT); first = false;
  if (content != kNone) L.str(content); else L.lit(S, EL_EMPTY_STR);
  if (task != kNone && L.slen(task) > 0) { L.lit(S, EL_TASK); L.str(task); }
  if (title != kNone) { L.lit(S, EL_TITLE); L.str(title); }
}

__device__ void el_item_instances(ElPlan& L, const ElShared& S, const ElItem& it, uint32_t gtask, bool& first) {
  const bool keep_title = it.task != kNone && it.title != kNone && L.slen(it.title) > 0 && L.str_is(it.task, "RETRIEVAL_DOCUMENT", 18);
  const uint32_t task = gtask != kNone ? gtask : it.task, title = keep_title ? it.title : kNone;
  if (L.W.ty(it.content) == T_QOPEN) el_instance(L, S, it.content, task, title, first);
  else if (L.W.ty(it.content + 1) != ']') for (uint32_t q = it.content + 1;;) {
    el_instance(L, S, L.is_null(q) ? kNone : q, task, title, first);
    const uint32_t nx = L.after(q);
    if (L.W.ty(nx) == ']') break;
    q = nx + 1;
  }
}

// the elements of array token a, in order: f(q) for each element token q; stops early when f returns non-zero (returned)
template <class F>
__device__ int el_each(const ElPlan& L, uint32_t a, F f) {
  if (L.W.ty(a + 1) == ']') return 0;
  for (uint32_t q = a + 1;;) {
    if (int r = f(q)) return r;
    const uint32_t nx = L.after(q);
    if (L.W.ty(nx) == ']') return 0;
    q = nx + 1;
  }
}

// plan_embeddings over the token view; returns the reason (0: OK, the ops planned) and fills res' model span / body_kind
__device__ int el_walk(ElPlan& L, ElShared& S, aigw_doc_result& res) {
  const EmbLargeParams& P = L.P;
  const ScanToks& W = L.W;
  const uint32_t ntok = W.ntok, dlb = S.dlb;
  const bool flat = dlb != kNone && !S.dnest;
  uint32_t input = kNone, model_raw = kNone, model = kNone, dims = kNone, autot = kNone, gtask = kNone;
  int prob = 0;
  bool syn = false;
  // ---- the root's members in body order (a syntax error anywhere wins over every problem)
  if (W.ty(0) == '{') {
    uint32_t seen = 0, j = 1;
    if (W.ty(1) == '}') j = 2;
    else for (;;) {
      if (W.ty(j) != T_QOPEN || W.ty(j + 1) != T_QCLOSE || W.ty(j + 2) != ':') { syn = true; break; }
      const uint32_t ko = W.ps(j) + 1u, kl = W.ps(j + 1) - ko;
      const bool kesc = W.has_backslash(ko, ko + kl);
      const uint8_t* kp = W.body + ko;
      const int slot = kesc ? -1 : scan_key_is(kp, kl, "input", 5) ? 0 : scan_key_is(kp, kl, "model", 5) ? 1 : scan_key_is(kp, kl, "encoding_format", 15) ? 2
                     : scan_key_is(kp, kl, "dimensions", 10) ? 3 : scan_key_is(kp, kl, "user", 4) ? 4 : scan_key_is(kp, kl, "auto_truncate", 13) ? 5
                     : scan_key_is(kp, kl, "task_type", 9) ? 6 : -1;
      int p = kesc ? AIGW_R_ESCAPE : 0;   // keys are compared raw here (documented in the header)
      if (slot >= 0) { if (seen & (1u << slot)) p = AIGW_R_DUP_KEY; seen |= 1u << slot; }
      const uint32_t v = j + 3;
      const uint32_t e = (v == dlb && flat) ? S.drb + 1u : L.after(v);
      if (e == kNone) { syn = true; break; }
      if (!p && slot >= 0) {
        const bool nul = L.is_null(v), str = W.ty(v) == T_QOPEN;
        switch (slot) {
          case 0: input = v; break;
          case 1: model_raw = v; if (!nul) { if (!str) p = AIGW_R_E400_TYPE; else model = v; } break;
          case 2: case 4: if (!nul && !str) p = AIGW_R_E400_TYPE; break;
          case 3: if (!nul) { p = emb_int_reason(W, v); dims = v; } break;
          case 5: if (!nul) { if (!L.is_bool(v)) p = AIGW_R_E400_TYPE; else autot = v; } break;
          case 6: if (!nul) { if (!str) p = AIGW_R_E400_TYPE; else if (L.slen(v) > 0) gtask = v; } break;
        }
      }
      if (p && !prob) prob = p;
      const uint32_t t2 = W.ty(e);
      j = e + 1u;
      if (t2 == ',') continue;
      if (t2 != '}') syn = true;
      break;
    }
    if (!syn && j != ntok) syn = true;   // bytes after the root
  } else {
    if (L.after(0) != ntok) syn = true;
    else if (!L.is_null(0)) prob = AIGW_R_E400_TYPE;
  }
  if (syn) return AIGW_R_E400_SYNTAX;
  if (prob) return prob;
  // ---- the input union: 0 none, 1 string, 2 []string, 3 item, 4 []item, 5 ints / int arrays
  int kind = 0;
  uint32_t count = 0;   // []string: elements
  if (input != kNone) {
    const uint32_t t = W.ty(input);
    if (t == T_QOPEN) kind = 1;
    else if (t == '{') { ElItem it; bool empty; if (int r = el_item(L, input, it, empty)) return r; if (empty) return AIGW_R_E400_CONTENT; kind = 3; }
    else if (t == '[') {
      const uint32_t f = input + 1, tf = W.ty(f);
      if (input == dlb && flat) {
        // checked in parallel: the first failing element in body order
        if (S.ifail != kNone) return (int)(S.ifail & 0xffu);
        kind = tf == ']' || tf == T_QOPEN ? 2 : 5;
        count = S.icount;
      } else if (tf == ']') kind = 2;
      else if (tf == T_QOPEN) {
        kind = 2;
        if (int r = el_each(L, input, [&](uint32_t q) { count++; return W.ty(q) != T_QOPEN && !L.is_null(q) ? AIGW_R_E400_TYPE : 0; })) return r;
      } else if (tf == '{') {
        kind = 4;
        if (int r = el_each(L, input, [&](uint32_t q) { ElItem it; bool empty; int x = el_item(L, q, it, empty); return x ? x : empty ? AIGW_R_E400_CONTENT : 0; })) return r;
      } else if (tf == '[') {
        kind = 5;
        if (int r = el_each(L, input, [&](uint32_t q) {
              if (L.is_null(q)) return 0;
              if (W.ty(q) != '[') return (int)AIGW_R_E400_TYPE;
              return el_each(L, q, [&](uint32_t x) { return L.is_null(x) ? 0 : emb_int_reason(W, x); });
            })) return r;
      } else if (L.is_num(f)) {
        kind = 5;
        if (int r = el_each(L, input, [&](uint32_t q) { return L.is_null(q) ? 0 : emb_int_reason(W, q); })) return r;
      } else return AIGW_R_E400_TYPE;
    } else return AIGW_R_E400_TYPE;
  }
  if (model != kNone) {
    const uint32_t mo = W.ps(model) + 1u, ml = L.slen(model);
    if (W.has_backslash(mo, mo + ml)) return AIGW_R_ESCAPE;
    if (ml > 0xffffu) return AIGW_R_TOO_LARGE;   // model_len is 16 bits
    res.model_off = mo; res.model_len = (uint16_t)ml;
  }
  const bool need_model = P.override_len != 0;
  if (need_model && !P.override_ok) return AIGW_R_UNSUPPORTED_FIELD;
  // ---- Amazon Titan through InvokeModel: one input text, optional dimensions
  if (P.base == AIGW_SCHEMA_AWS_BEDROCK) {
    uint32_t text = kNone;
    if (kind == 1) text = input;
    else if (kind == 2) { if (count != 1) return AIGW_R_E422_CONTENT; if (!L.is_null(input + 1)) text = input + 1; }
    else return AIGW_R_E422_CONTENT;
    // :path = /model/<url.PathEscape(model)>/invoke, the escaped model in the CTA's scratch
    const uint8_t* mp = (const uint8_t*)P.override_model;
    uint32_t ml = P.override_len;
    if (!need_model) { mp = model != kNone ? W.body + W.ps(model) + 1u : nullptr; ml = model != kNone ? L.slen(model) : 0u; }
    uint32_t sw = 0;
    for (uint32_t i = 0; i < ml; i++) {
      const uint32_t c = mp[i];
      const bool keep = (c - 'a' < 26u) || (c - 'A' < 26u) || (c - '0' < 10u) || c == '-' || c == '_' || c == '.' || c == '~' || c == '$' || c == '&' ||
                        c == '+' || c == ':' || c == '=' || c == '@';
      if (sw + 3u > kEmbScratch - 64u) return AIGW_R_TOO_LARGE;
      if (keep) L.w.scr[sw++] = (uint8_t)c;
      else { const char* hx = "0123456789ABCDEF"; L.w.scr[sw++] = '%'; L.w.scr[sw++] = (uint8_t)hx[c >> 4]; L.w.scr[sw++] = (uint8_t)hx[c & 15u]; }
    }
    L.lit(S, EL_PATH_MODEL);
    if (sw) { L.push(OP_SCR, 0, sw); L.olen += sw; }
    L.lit(S, EL_INVOKE);
    if (L.olen > 0xffffu) return AIGW_R_TOO_LARGE;   // path_len is 16 bits
    S.path_len = L.olen;
    res.body_kind = AIGW_BODY_BYTES;
    L.lit(S, EL_TITAN_OPEN);
    if (text == kNone) L.lit(S, EL_EMPTY_STR); else L.str(text);
    if (dims != kNone) { L.lit(S, EL_TITAN_DIMS); L.span(W.ps(dims), W.scalar_end(dims) - W.ps(dims)); }
    L.lit(S, EL_RBRACE);
    return L.err;
  }
  // ---- :path
  if (P.base == AIGW_SCHEMA_OPENAI) L.lit(S, EL_OPENAI_PATH);
  else {
    L.lit(S, P.base == AIGW_SCHEMA_AZURE_OPENAI ? EL_AZ_PATH1 : EL_GOOGLE_PATH);
    if (need_model) L.lit(S, EL_OVERRIDE); else if (model != kNone) L.span(W.ps(model) + 1u, L.slen(model));
    if (P.base == AIGW_SCHEMA_AZURE_OPENAI) { L.lit(S, EL_AZ_PATH2); L.lit(S, EL_VERSION); } else L.lit(S, EL_PREDICT);
  }
  if (L.olen > 0xffffu) return AIGW_R_TOO_LARGE;   // path_len is 16 bits
  S.path_len = L.olen;
  if (P.base != AIGW_SCHEMA_GCP_VERTEX) {
    // sjson.SetBytesOptions(original, "model", override): splice the first "model" value, or append the member at the root
    if (!need_model) { if (P.force_mutation) { L.span(0, W.len); res.body_kind = AIGW_BODY_BYTES; } return L.err; }
    res.body_kind = AIGW_BODY_BYTES;
    if (W.ty(0) != '{') {   // a null root
      L.lit(S, EL_LBRACE); L.lit(S, EL_MODEL_MEMBER); L.lit(S, EL_QUOTE); L.lit(S, EL_OVERRIDE); L.lit(S, EL_QUOTE); L.lit(S, EL_RBRACE);
    } else if (model_raw != kNone) {
      const uint32_t b = W.ps(model_raw), e = W.ty(model_raw) == T_QOPEN ? W.ps(model_raw + 1) + 1u : W.scalar_end(model_raw);
      L.span(0, b); L.lit(S, EL_QUOTE); L.lit(S, EL_OVERRIDE); L.lit(S, EL_QUOTE); L.span(e, W.len - e);
    } else {
      const uint32_t o = W.ps(0), c = W.ps(ntok - 1);
      L.span(o, c - o); if (ntok != 2) L.lit(S, EL_COMMA);
      L.lit(S, EL_MODEL_MEMBER); L.lit(S, EL_QUOTE); L.lit(S, EL_OVERRIDE); L.lit(S, EL_QUOTE); L.lit(S, EL_RBRACE);
    }
    return L.err;
  }
  // ---- Vertex: gcp.PredictRequest{instances, parameters}
  if (kind == 0 || kind == 5) return AIGW_R_E500_ARGS;   // "unsupported input type for embedding"
  res.body_kind = AIGW_BODY_BYTES;
  L.lit(S, EL_INSTANCES);
  if (kind == 2 && W.ty(input + 1) == ']') L.lit(S, EL_NULL);
  else {
    bool first = true;
    L.lit(S, EL_LBRACK);
    if (kind == 1) el_instance(L, S, input, gtask, kNone, first);
    else if (kind == 2) {
      if (input == dlb && flat) {   // strings and nulls, commas between
        for (uint32_t q = input + 1; q < S.drb; q += W.ty(q) == T_QOPEN ? 3u : 2u) { el_instance(L, S, L.is_null(q) ? kNone : q, gtask, kNone, first); if (L.err) break; }
      } else el_each(L, input, [&](uint32_t q) { el_instance(L, S, L.is_null(q) ? kNone : q, gtask, kNone, first); return L.err; });
    } else if (kind == 3) { ElItem it; bool e2; el_item(L, input, it, e2); el_item_instances(L, S, it, gtask, first); }
    else el_each(L, input, [&](uint32_t q) { ElItem it; bool e2; el_item(L, q, it, e2); el_item_instances(L, S, it, gtask, first); return L.err; });
    L.lit(S, EL_LAST);
  }
  L.lit(S, EL_PARAMS);
  bool pf = true;
  if (autot != kNone && W.body[W.ps(autot)] == 't') { L.lit(S, EL_AUTOTRUNC); pf = false; }
  if (dims != kNone) {
    const uint32_t o = W.ps(dims), e = W.scalar_end(dims);
    bool pos = W.body[o] != '-';
    if (pos) { pos = false; for (uint32_t i = o; i < e; i++) if (W.body[i] != '0') pos = true; }
    if (pos) { if (!pf) L.lit(S, EL_COMMA); L.lit(S, EL_DIMS); L.span(o, e - o); }
  }
  L.lit(S, EL_END);
  return L.err;
}

// ---------------------------------------------------------------- emit
struct ElEsc {
  const uint4* e; uint32_t ne, dtotal;
  __device__ uint32_t pos(uint32_t k) const { return e[k].x & 0xffffffu; }
  __device__ uint32_t in(uint32_t k) const { return (e[k].x >> 24) & 15u; }
  __device__ uint32_t out(uint32_t k) const { return e[k].x >> 28; }
  __device__ uint32_t D(uint32_t k) const { return k < ne ? e[k].w : dtotal; }   // sum of (in - out) over the entries before k (mod 2^32)
  __device__ uint32_t byte(uint32_t k, uint32_t t) const { return t < 4u ? (e[k].y >> (8u * t)) & 255u : (e[k].z >> (8u * (t - 4u))) & 255u; }
  __device__ uint32_t lower(uint32_t p) const {   // first entry at or after position p
    uint32_t lo = 0, hi = ne;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (pos(m) < p) lo = m + 1; else hi = m; }
    return lo;
  }
};

// a sequential reader of the record's bytes from output offset o on: op k, and inside an emitted string the next escape entry
struct ElCursor {
  const uint4* ops; uint32_t nops; const ElEsc& E; const uint8_t* body; const uint8_t* lits; const uint8_t* scr;
  uint32_t k, kind, a, y, end, ea;   // the op in hand
  uint32_t ip, ke, eo;               // input (or literal / scratch) position; STR: next entry, offset in it (kNone: not inside)

  __device__ ElCursor(const uint4* o, uint32_t n, const ElEsc& e, const uint8_t* b, const uint8_t* l, const uint8_t* s) : ops(o), nops(n), E(e), body(b), lits(l), scr(s) {}
  __device__ void load(uint32_t kk) { k = kk; const uint4 v = ops[kk]; kind = v.x >> 29; a = v.x & 0x1fffffffu; y = v.y; end = v.z; ea = v.w; }
  __device__ uint32_t start() const { return k ? ops[k - 1].z : 0u; }
  // out position of entry j inside the string of this op
  __device__ uint32_t opos(uint32_t j) const { return (E.pos(j) - a) - (E.D(j) - E.D(ea)); }
  __device__ void seek(uint32_t r) {   // r: offset inside op k
    eo = kNone;
    if (kind != OP_STR) { ip = kind == OP_LIT ? (a & 0xffffu) + r : a + r; return; }
    // last entry j >= ea with opos(j) <= r (opos grows with j, and entries past the string have opos beyond its length)
    uint32_t lo = ea, hi = E.ne;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (opos(m) <= r) lo = m + 1; else hi = m; }
    if (lo == ea) { ip = a + r; ke = ea; return; }
    const uint32_t j = lo - 1u, op = opos(j);
    if (r < op + E.out(j)) { ke = j; eo = r - op; return; }
    ip = E.pos(j) + E.in(j) + (r - op - E.out(j)); ke = j + 1u;
  }
  __device__ void at(uint32_t o) {
    uint32_t lo = 0, hi = nops;
    while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if (ops[m].z <= o) lo = m + 1; else hi = m; }
    load(lo); seek(o - start());
  }
  __device__ uint32_t next(uint32_t o) {   // the byte at output offset o (the one after the previous call's)
    while (o >= end) { load(k + 1u); seek(0); }
    if (kind == OP_LIT) return lits[ip++];
    if (kind == OP_SCR) return scr[ip++];
    if (kind == OP_SPAN) return body[ip++];
    if (eo == kNone && ke < E.ne && E.pos(ke) == ip) eo = 0;
    if (eo == kNone) return body[ip++];
    const uint32_t c = E.byte(ke, eo);
    if (++eo == E.out(ke)) { ip = E.pos(ke) + E.in(ke); ke++; eo = kNone; }
    return c;
  }
};

__global__ void __launch_bounds__(kElThreads, 2) emb_large_kernel(const __grid_constant__ EmbLargeParams P) {
  __shared__ ElShared S;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
  const uint32_t lt = (1u << lane) - 1u;
  uint8_t* slice = P.ws + (size_t)blockIdx.x * P.slice;
  ElWork wk;
  wk.tok = (uint32_t*)slice;
  wk.esc = (uint4*)(slice + (((size_t)P.tok_cap * 4u + 15u) & ~(size_t)15u));   // 16-byte aligned: entries are read as uint4
  wk.ops = wk.esc + P.esc_cap;
  wk.dep = (uint8_t*)(wk.ops + P.op_cap);
  wk.scr = wk.dep + (((size_t)P.tok_cap + 15u) & ~(size_t)15u);
  for (uint32_t k = tid; k < sizeof S.lits; k += kElThreads) S.lits[k] = (uint8_t)P.lits[k];
  for (uint32_t k = tid; k < EL_COUNT; k += kElThreads) { S.lit_off[k] = P.lit_off[k]; S.lit_len[k] = P.lit_len[k]; }
  const bool respell = P.base == AIGW_SCHEMA_GCP_VERTEX || P.base == AIGW_SCHEMA_AWS_BEDROCK;
  for (;;) {
    __syncthreads();
    if (tid == 0) {
      S.doc = atomicAdd(P.next, 1u); S.fail = kNone; S.dlb = S.drb = kNone; S.dnest = S.dsyn = 0; S.ifail = kNone; S.icount = 0;
      S.nops = 0; S.path_len = 0; S.total = 0; S.dtotal = 0; S.off = ~0ull;
    }
    __syncthreads();
    const uint32_t doc = S.doc;
    if (doc >= P.n) break;
    const uint8_t* body = P.bodies + P.offsets[doc];
    const uint32_t len = P.lens[doc];
    const uint32_t cap = min(emb_tok_cap(len), P.tok_cap), ecap = min(emb_esc_cap(len), P.esc_cap);
    int fail = 0;
    uint32_t ntok = 0, ne = 0;
    if (P.call_reason) fail = (int)P.call_reason;
    else if (len >= (1u << 24) || len == 0) fail = len ? AIGW_R_TOO_LARGE : AIGW_R_E400_SYNTAX;
    else if (((uintptr_t)body) & 15u) fail = AIGW_R_ARGS;   // the arena convention: every request starts 16-byte aligned
    uint32_t in_str = 0, prev_sc = 0, esc_c = 0, prev_em = 0;   // carries across tiles (uniform over the CTA)
    uint4 na = make_uint4(0, 0, 0, 0), nb = na;
    if (!fail && tid * 32u + 32u <= len) { na = __ldg((const uint4*)(body + tid * 32u)); nb = __ldg((const uint4*)(body + tid * 32u + 16)); }
    // ================================================================ scan
    if (!fail) for (uint32_t base = 0, it = 0; base < len; base += kElTile, it ^= 1u) {
      const uint32_t pos0 = base + tid * 32u;
      uint32_t w[8];
      if (pos0 + 32u <= len) {
        w[0] = na.x; w[1] = na.y; w[2] = na.z; w[3] = na.w; w[4] = nb.x; w[5] = nb.y; w[6] = nb.z; w[7] = nb.w;
        if (pos0 + kElTile + 32u <= len) { na = __ldg((const uint4*)(body + pos0 + kElTile)); nb = __ldg((const uint4*)(body + pos0 + kElTile + 16)); }
      } else {
#pragma unroll
        for (int k = 0; k < 8; k++) {   // past the end: spaces, which are no token and no escape
          uint32_t v = 0x20202020u;
          const uint32_t p = pos0 + 4u * k;
          if (p + 4u <= len) v = __ldg((const uint32_t*)(body + p));
          else if (p < len) { v = 0; for (uint32_t q = 0; q < 4; q++) v |= (uint32_t)(p + q < len ? body[p + q] : 0x20u) << (8u * q); }
          w[k] = v;
        }
      }
      const ByteClasses c = classify32(w);
      // ---- escapes: carry-in from the nearest preceding thread that is not all backslashes
      const uint32_t bsm = c.bslash;
      const bool allbs = bsm == FULL;
      const uint32_t tpar = __clz(~bsm) & 1u;
      const uint32_t nbm = __ballot_sync(FULL, !allbs);
      const uint32_t below = nbm & lt;
      const uint32_t lane_c = __shfl_sync(FULL, tpar, below ? 31u - __clz(below) : 0u);
      const uint32_t warp_c = __shfl_sync(FULL, tpar, nbm ? 31u - __clz(nbm) : 0u);
      if (lane == 0) S.wesc[it][warp] = nbm ? 2u | warp_c : 0u;
      __syncthreads();
      uint32_t cin_w = esc_c, cout_t = esc_c;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t e = S.wesc[it][k]; if (e) { if (k < warp) cin_w = e & 1u; cout_t = e & 1u; } }
      const uint32_t cin = below ? lane_c : cin_w;
      const uint32_t esc = bsm | cin ? escaped_mask(bsm, cin) & (pos0 >= len ? 0u : pos0 + 32u <= len ? FULL : (1u << (len - pos0)) - 1u) : 0u;
      // ---- string parity of the unescaped quotes
      const uint32_t uq = c.quote & ~esc;
      const uint32_t bal = __ballot_sync(FULL, (__popc(uq) & 1u) != 0);
      if (lane == 0) S.wpar[it][warp] = __popc(bal) & 1u;
      if (lane == 31) S.wem[it][warp] = esc;   // the escaped bytes of the warp's last thread: the next thread's low-surrogate check
      __syncthreads();
      uint32_t pre = 0, tot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wpar[it][k]; tot ^= v; if (k < warp) pre ^= v; }
      const uint32_t in0 = in_str ^ pre ^ (__popc(bal & lt) & 1u);
      const uint32_t ps = prefix_xor32(uq) ^ (in0 ? FULL : 0u);
      const uint32_t inside = ps & ~uq;
      const uint32_t out = ~ps & ~uq;
      if (c.ctl & inside) raise_min(fail, AIGW_R_CTRL_IN_STRING);
      if ((c.ctl & out & ~c.ws) || (bsm & out)) raise_min(fail, AIGW_R_E400_SYNTAX);
      uint32_t ecnt = 0;
      for (uint32_t e = esc & inside; e;) {
        const uint32_t i = __ffs(e) - 1u; e &= e - 1u;
        const uint32_t p = pos0 + i, ch = body[p];
        const bool ok = ch == '"' || ch == '\\' || ch == '/' || ch == 'b' || ch == 'f' || ch == 'n' || ch == 'r' || ch == 't' ||
                        (ch == 'u' && p + 4u < len && is_hex(body[p + 1]) && is_hex(body[p + 2]) && is_hex(body[p + 3]) && is_hex(body[p + 4]));
        if (!ok) raise_min(fail, AIGW_R_ESCAPE);
        else if (respell && (ch == '/' || ch == 'b' || ch == 'f' || ch == 'u')) ecnt++;   // an upper bound: pairs' low halves drop out below
      }
      const uint32_t up_esc = __shfl_up_sync(FULL, esc, 1);
      const uint32_t pesc = lane ? up_esc : warp ? S.wem[it][warp - 1] : prev_em;   // the previous thread's escaped bytes
      // ---- tokens (low 16 bits) and escape entries (high 16 bits), compacted together
      const uint32_t sc = out & ~c.op & ~c.ws;
      if (lane == 31) S.wlast[it][warp] = sc >> 31;
      uint32_t prev = __shfl_up_sync(FULL, sc >> 31, 1);
      const uint32_t last_em_tile = S.wem[it][7];
      __syncthreads();
      if (lane == 0) prev = warp == 0 ? prev_sc : S.wlast[it][warp - 1];
      const uint32_t sc_start = sc & ~((sc << 1) | prev);
      uint32_t tk = (c.op & out) | uq | sc_start;
      // the exact entry count: drop the low halves of surrogate pairs
      auto is_esc = [&](uint32_t q) -> bool { return q >= pos0 ? (esc >> (q - pos0)) & 1u : q + 32u >= pos0 ? (pesc >> (q + 32u - pos0)) & 1u : false; };
      if (ecnt) {
        ecnt = 0;
        for (uint32_t e = esc & inside; e;) {
          const uint32_t i = __ffs(e) - 1u; e &= e - 1u;
          uint4 en;
          if (respell && esc_entry(body, len, pos0 + i, is_esc, en)) ecnt++;
        }
      }
      const uint32_t cnt = __popc(tk) | (ecnt << 16);
      uint32_t incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) { const uint32_t v = __shfl_up_sync(FULL, incl, d); if ((int)lane >= d) incl += v; }
      if (lane == 31) S.wcnt[it][warp] = incl;
      const uint32_t last_sc_tile = S.wlast[it][7];
      __syncthreads();
      uint32_t wpre = 0, wtot = 0;
#pragma unroll
      for (uint32_t k = 0; k < 8; k++) { const uint32_t v = S.wcnt[it][k]; wtot += v; if (k < warp) wpre += v; }
      const uint32_t ex = wpre + incl - cnt;
      uint32_t off = ntok + (ex & 0xffffu);
      while (tk) {
        const uint32_t i = __ffs(tk) - 1u; tk &= tk - 1u;
        const uint32_t p = pos0 + i, bit = 1u << i;
        const uint32_t ty = (uq & bit) ? ((ps & bit) ? T_QOPEN : T_QCLOSE) : (c.op & bit) ? (uint32_t)body[p] : T_SCALAR;
        if (off < cap) wk.tok[off] = p | (ty << 24);
        off++;
      }
      if (ecnt) {
        uint32_t eoff = ne + (ex >> 16);
        for (uint32_t e = esc & inside; e;) {
          const uint32_t i = __ffs(e) - 1u; e &= e - 1u;
          uint4 en;
          if (esc_entry(body, len, pos0 + i, is_esc, en)) { if (eoff < ecap) wk.esc[eoff] = en; eoff++; }
        }
      }
      ntok += wtot & 0xffffu; ne += wtot >> 16; in_str ^= tot; prev_sc = last_sc_tile; esc_c = cout_t; prev_em = last_em_tile;
    }
    if (!fail && in_str) fail = AIGW_R_E400_SYNTAX;   // unterminated string
    if (ntok > cap) raise_min(fail, AIGW_R_TOKENS);
    if (ne > ecap) raise_min(fail, AIGW_R_SCRATCH);
    if (!fail && ntok == 0) fail = AIGW_R_E400_SYNTAX;   // white space only
    if (fail) atomicMin(&S.fail, (uint32_t)fail);
    __syncthreads();
    const ScanToks W{wk.tok, ntok, body, len};
    // ================================================================ depth, scalar grammar, the root's "input" array
    if (S.fail == kNone) {
      int carry = 0;
      uint32_t it = 0;
      for (uint32_t b0 = 0; b0 < ntok; b0 += kElThreads, it ^= 1u) {
        const uint32_t j = b0 + tid;
        const uint32_t ty = j < ntok ? wk.tok[j] >> 24 : 0u;
        const int d = (ty == '{' || ty == '[') ? 1 : (ty == '}' || ty == ']') ? -1 : 0;
        uint32_t tot;
        const int da = carry + (int)block_excl<uint32_t>((uint32_t)d, S.wsum, it, tot) + d;
        carry += (int)tot;
        if (j < ntok) {
          if (da < 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
          else if (da > (int)kEmbMaxDepth) atomicMin(&S.fail, (uint32_t)AIGW_R_DEPTH);
          wk.dep[j] = (uint8_t)(da < 0 ? 0 : da > 127 ? 127 : da);
          if (ty == T_SCALAR && !W.scalar_kind(j)) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
          if (ty == '[' && da == 2 && j >= 4 && (wk.tok[j - 1] >> 24) == ':' && (wk.tok[j - 2] >> 24) == T_QCLOSE && (wk.tok[j - 3] >> 24) == T_QOPEN) {
            const uint32_t o = (wk.tok[j - 3] & 0xffffffu) + 1u;
            if (scan_key_is(body + o, (wk.tok[j - 2] & 0xffffffu) - o, "input", 5)) atomicMin(&S.dlb, j);
          }
        }
      }
      if (carry != 0 && tid == 0) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
    }
    // the escape list's width changes: exclusive prefix sum into each entry's w (only for a request still in play, whose entries
    // all fit the slice)
    __syncthreads();   // the depth pass's last round has read S.wsum, and its failures are in S.fail
    if (ne && ne <= ecap && S.fail == kNone) {
      uint32_t run = 0, it = 0;
      for (uint32_t b0 = 0; b0 < ne; b0 += kElThreads, it ^= 1u) {
        const uint32_t k = b0 + tid;
        uint4 en = k < ne ? wk.esc[k] : make_uint4(0, 0, 0, 0);
        const uint32_t d = k < ne ? ((en.x >> 24) & 15u) - (en.x >> 28) : 0u;
        uint32_t tot;
        const uint32_t ex = block_excl<uint32_t>(d, S.wsum, it, tot);
        if (k < ne) wk.esc[k].w = run + ex;
        run += tot;
      }
      if (tid == 0) S.dtotal = run;
    }
    __syncthreads();
    // ================================================================ a flat input array, in parallel
    const uint32_t dlb = S.dlb;
    if (S.fail == kNone && dlb != kNone) {
      for (uint32_t j = dlb + 1u + tid; j < ntok; j += kElThreads) {
        const uint32_t ty = wk.tok[j] >> 24;
        if ((ty == ']' || ty == '}') && wk.dep[j] == 1) atomicMin(&S.drb, j);
      }
      __syncthreads();
      const uint32_t drb = S.drb;
      if (drb == kNone || (wk.tok[drb] >> 24) != ']') { if (tid == 0) S.dnest = 1; }
      else {
        const uint32_t t0 = wk.tok[dlb + 1] >> 24;
        // the union's form, from the first element: 0 empty / bad first, 1 strings, 2 ints, 3 arrays of ints
        const int form = dlb + 1u == drb ? 0 : t0 == T_QOPEN ? 1 : t0 == '[' ? 3 : (t0 == T_SCALAR && (body[wk.tok[dlb + 1] & 0xffffffu] == '-' || (body[wk.tok[dlb + 1] & 0xffffffu] - '0') < 10u)) ? 2 : 0;
        if (tid == 0 && dlb + 1u != drb && form == 0) atomicMin(&S.ifail, ((dlb + 1u) << 8) | AIGW_R_E400_TYPE);
        uint32_t nel = 0;
        for (uint32_t j = dlb + 1u + tid; j < drb; j += kElThreads) {
          const uint32_t ty = wk.tok[j] >> 24, pv = wk.tok[j - 1] >> 24, nx = wk.tok[j + 1] >> 24;
          const uint32_t dj = wk.dep[j] & 0x7fu;
          bool syn = false;
          if (ty == '{' || ty == '}' || ty == ':') { S.dnest = 1; continue; }
          const bool vstart_prev = pv == '[' || pv == ',';
          const bool vend_next = nx == ',' || nx == ']';
          if (ty == T_QOPEN) syn = !vstart_prev || nx != T_QCLOSE;
          else if (ty == T_QCLOSE) syn = !vend_next;
          else if (ty == T_SCALAR) syn = !vstart_prev || !vend_next;
          else if (ty == '[') syn = !vstart_prev || !(nx == T_QOPEN || nx == T_SCALAR || nx == '[' || nx == ']');
          else if (ty == ']') syn = !(pv == T_QCLOSE || pv == T_SCALAR || pv == ']' || pv == '[') || !vend_next;
          else if (ty == ',') syn = !(pv == T_QCLOSE || pv == T_SCALAR || pv == ']') || !(nx == T_QOPEN || nx == T_SCALAR || nx == '[');
          if (syn) { S.dsyn = 1; continue; }
          // the element's level: value starts at depth 2 are elements, at depth 3 the elements of an element array
          const bool vstart = ty == T_QOPEN || ty == T_SCALAR || ty == '[';
          if (!vstart) continue;
          const uint32_t lvl = ty == '[' ? dj - 1u : dj;   // depth before the token
          int r = 0;
          const bool nul = ty == T_SCALAR && body[wk.tok[j] & 0xffffffu] == 'n';
          if (lvl == 2) {
            nel++;
            if (form == 1) r = ty == T_QOPEN || nul ? 0 : AIGW_R_E400_TYPE;
            else if (form == 2) r = nul ? 0 : emb_int_reason(W, j);
            else if (form == 3) r = nul || ty == '[' ? 0 : AIGW_R_E400_TYPE;
          } else if (lvl == 3 && form == 3) r = nul ? 0 : emb_int_reason(W, j);
          if (r) atomicMin(&S.ifail, (j << 8) | (uint32_t)r);
        }
        if (nel) atomicAdd(&S.icount, nel);
      }
      __syncthreads();
      if (tid == 0 && !S.dnest && S.dsyn) atomicMin(&S.fail, (uint32_t)AIGW_R_E400_SYNTAX);
    }
    __syncthreads();
    // ================================================================ the members, the plan
    if (tid == 0) {
      aigw_doc_result res;
      res.out_off = 0; res.body_len = 0; res.path_len = 0; res.status = AIGW_DECLINED; res.reason = 0; res.model_off = 0; res.model_len = 0;
      res.body_kind = AIGW_BODY_UNCHANGED; res.flags = 0; res.in_len = len; res._pad = 0;
      int f = S.fail == kNone ? 0 : (int)S.fail;
      uint32_t nops = 0;
      if (!f) {
        ElPlan L(P, W, wk);
        f = el_walk(L, S, res);
        nops = L.nops;
      }
      if (f) { res.model_off = 0; res.model_len = 0; res.body_kind = AIGW_BODY_UNCHANGED; nops = 0; }
      S.nops = nops;
      S.res = res;
      S.fail = f ? (uint32_t)f : kNone;
    }
    __syncthreads();
    if (S.fail != kNone) {
      if (tid == 0) {
        aigw_doc_result res = S.res;
        const int f = (int)S.fail;
        res.reason = (uint8_t)f; res.status = f >= 48 ? AIGW_INTERNAL : f >= 40 ? AIGW_INVALID_422 : f >= 32 ? AIGW_MALFORMED_400 : AIGW_DECLINED;
        P.results[doc] = res;
      }
      continue;
    }
    // ================================================================ op lengths, prefix sum, a lone surrogate in an emitted string
    const ElEsc E{wk.esc, ne, S.dtotal};
    const uint32_t nops = S.nops;
    {
      // Lengths add up in 64 bits: a long request-level task_type repeated for a million null inputs asks for terabytes.  The
      // op ends are saturated just above the ceiling (below 2^32), which keeps them ordered; such a record is declined below.
      const unsigned long long lim = emb_out_ceiling(len) + 1u;
      unsigned long long run = 0;
      uint32_t it = 0;
      for (uint32_t b0 = 0; b0 < nops; b0 += kElThreads, it ^= 1u) {
        const uint32_t k = b0 + tid;
        uint32_t n = 0;
        if (k < nops) {
          uint4 op = wk.ops[k];
          const uint32_t kind = op.x >> 29;
          if (kind == OP_STR) {
            const uint32_t q0 = op.x & 0x1fffffffu, q1 = op.y;
            const uint32_t ea = E.lower(q0), eb = E.lower(q1);
            n = (q1 + 1u - q0) - (E.D(eb) - E.D(ea));
            op.w = ea;
          } else n = op.y;
          wk.ops[k] = op;
        }
        unsigned long long tot;
        const unsigned long long ex = block_excl<unsigned long long>(n, S.wsum64, it, tot);
        if (k < nops) wk.ops[k].z = (uint32_t)min(run + ex + n, lim);
        run += tot;
      }
      if (tid == 0) S.total = run;
      for (uint32_t k = tid; k < ne; k += kElThreads) {
        if (E.in(k) == 6u && E.out(k) == 15u) {
          // the string around a lone surrogate: the last token at or before it is its opening quote
          const uint32_t p = E.pos(k);
          uint32_t lo = 0, hi = ntok;
          while (lo < hi) { const uint32_t m = (lo + hi) >> 1; if ((wk.tok[m] & 0xffffffu) <= p) lo = m + 1; else hi = m; }
          if (lo && (wk.dep[lo - 1] & 0x80u)) atomicMin(&S.fail, (uint32_t)AIGW_R_ESCAPE);
        }
      }
    }
    __syncthreads();
    if (tid == 0) {
      aigw_doc_result res = S.res;
      const unsigned long long total = S.total;
      int f = S.fail == kNone ? 0 : (int)S.fail;
      if (!f && total > emb_out_ceiling(len)) f = AIGW_R_OUT_SPACE;   // body_len stays 0: no arena takes it
      if (!f) {
        const unsigned long long size = ((unsigned long long)total + 15u) & ~15ull;
        const unsigned long long o = atomicAdd(P.out_used, size);
        if (o + size > P.out_capacity) { f = AIGW_R_OUT_SPACE; res.body_len = (uint32_t)total; }   // the record length this request needs
        else { S.off = o; res.out_off = o; res.path_len = (uint16_t)S.path_len; res.body_len = (uint32_t)total - S.path_len; res.status = AIGW_OK; }
      }
      if (f) {
        res.status = AIGW_DECLINED; res.reason = (uint8_t)f; res.path_len = 0; res.body_kind = AIGW_BODY_UNCHANGED; res.model_off = 0; res.model_len = 0;
        if (f != AIGW_R_OUT_SPACE) res.body_len = 0;
      }
      P.results[doc] = res;
    }
    __syncthreads();
    if (S.off == ~0ull) continue;
    // ================================================================ emit: 16-byte chunks, every thread busy
    const uint32_t total = (uint32_t)S.total, nchunk = (total + 15u) >> 4;   // at most the ceiling here
    uint4* dst = (uint4*)(P.out + S.off);
    ElCursor cur(wk.ops, nops, E, body, S.lits, wk.scr);
    for (uint32_t c = tid; c < nchunk; c += kElThreads) {
      const uint32_t o0 = c << 4;
      cur.at(o0);
      uint4 v;
      const bool one_op = o0 + 16u <= cur.end;
      if (one_op && cur.kind == OP_SPAN) v = load16_unaligned(body + cur.ip);
      else if (one_op && cur.kind == OP_STR && cur.eo == kNone && (cur.ke >= ne || E.pos(cur.ke) >= cur.ip + 16u)) v = load16_unaligned(body + cur.ip);
      else {
        unsigned long long lo = 0, hi = 0;   // zero past the record's end
        for (uint32_t b = 0; b < 16u && o0 + b < total; b++) {
          const unsigned long long x = cur.next(o0 + b);
          if (b < 8u) lo |= x << (8u * b); else hi |= x << (8u * (b - 8u));
        }
        v = make_uint4((uint32_t)lo, (uint32_t)(lo >> 32), (uint32_t)hi, (uint32_t)(hi >> 32));
      }
      dst[c] = v;
    }
  }
}

uint64_t emb_large_slice_bytes(uint32_t max_len) {
  const uint64_t tc = emb_tok_cap(max_len), ec = emb_esc_cap(max_len), oc = emb_op_cap(max_len);
  return ((((tc * 4u + 15u) & ~15ull) + ec * 16u + oc * 16u + ((tc + 15u) & ~15ull) + kEmbScratch) + 255u) & ~255ull;
}

int emb_large_grid(int sm_count, uint32_t max_len) {
  uint64_t g = kElWorkspace / emb_large_slice_bytes(max_len);
  if (g > (uint64_t)sm_count * 2u) g = (uint64_t)sm_count * 2u;
  return g < 1 ? 1 : (int)g;
}

void emb_large_lits(EmbLargeParams& P, const char* openai_path, uint32_t path_len, const char* override_model, uint32_t override_len,
                    const char* version, uint32_t version_len) {
  static const char* const kText[EL_OPENAI_PATH] = {
      "{\"instances\":", "{\"content\":", "},{\"content\":", ",\"task_type\":", ",\"title\":", "}]", ",\"parameters\":{", "\"auto_truncate\":true",
      "\"outputDimensionality\":", "}}", "publishers/google/models/", ":predict", "/openai/deployments/", "/embeddings?api-version=", "{\"inputText\":",
      ",\"dimensions\":", "/model/", "/invoke", "null", "\"\"", ",", "\"model\":", "\"", "{", "}", "["};
  uint32_t at = 0;
  auto put = [&](uint32_t id, const char* s, uint32_t n) { P.lit_off[id] = (uint16_t)at; P.lit_len[id] = (uint16_t)n; memcpy(P.lits + at, s, n); at += n; };
  memset(P.lits, 0, sizeof P.lits);
  for (uint32_t i = 0; i < EL_OPENAI_PATH; i++) put(i, kText[i], (uint32_t)strlen(kText[i]));
  put(EL_OPENAI_PATH, openai_path, path_len);
  put(EL_OVERRIDE, override_model, override_len);
  put(EL_VERSION, version, version_len);
  memset(P.override_model, 0, sizeof P.override_model);
  memcpy(P.override_model, override_model, override_len);
}

cudaError_t launch_emb_large(const EmbLargeParams& P, int grid, cudaStream_t st) {
  emb_large_kernel<<<P.n < (uint32_t)grid ? (P.n ? P.n : 1u) : (uint32_t)grid, kElThreads, 0, st>>>(P);
  return cudaGetLastError();
}

}  // namespace aigw
