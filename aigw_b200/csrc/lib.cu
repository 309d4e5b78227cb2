// aigw_b200 C-ABI implementation: context, arenas, device- and host-buffer entry points.
// The host path is a 3-slot pipeline: H2D(chunk c+1) ‖ kernel(chunk c) ‖ D2H(chunk c-1) on three
// CUDA streams; everything computed is computed by the kernels in this directory — there is no
// CPU fallback anywhere in this library.
#include <chrono>
#include <cstdio>
#include <sched.h>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <string>
#include <thread>
#include <type_traits>
#include <vector>

#include "chat_kernel.cuh"
#include "lib_internal.h"
#include "sse_kernel.cuh"
#include "bedrock_stream_kernel.cuh"
#include "mutate_kernel.cuh"
#include "sha256_kernel.cuh"
#include "cel_kernel.cuh"
#include "stream_kernel.cuh"
#include "bpe_kernel.cuh"
#include "emb_kernel.cuh"
#include "rerank_large_kernel.cuh"
#include "emb_large_kernel.cuh"
#include "chat_large_kernel.cuh"
#include "chat_bedrock_large_kernel.cuh"
#include "chat_anthropic_large_kernel.cuh"
#include "chat_gemini_large_kernel.cuh"
#include "messages_large_kernel.cuh"
#include "responses_large_kernel.cuh"
#include "completions_large_kernel.cuh"

#include <mutex>

using namespace aigw;

struct aigw_cost_program {
  aigw::CelProgramHost h;
  ~aigw_cost_program() { cudaFree(h.d_code); cudaFree(h.d_strings); }   // on the current device, like Scratch
};

// a failed call is reported once: its code is also taken off the thread's "last error", so that the launch check of a later call does not find it
#define CK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) { ctx->err = std::string(#x) + ": " + cudaGetErrorString(_e); (void)cudaGetLastError(); return (int)_e; } } while (0)
// Prologue of every int-returning C-ABI call that reaches the GPU: the context's device becomes current, checked like any other call
// (a thread may have made another GPU current since the last call).  ENTER_ON also names the stream the call runs on: the caller's,
// or the context's compute stream when the caller passes none.
#define ENTER() CK(cudaSetDevice(ctx->device))
#define ENTER_ON(stream) ENTER(); const cudaStream_t st = (stream) ? (cudaStream_t)(stream) : ctx->s_compute

// An owning, grow-only scratch buffer of device memory or, Pinned, of mapped pinned host memory.  ensure(bytes) keeps it at least
// `bytes` long: a shorter buffer is freed and reallocated with headroom (bytes + bytes/8 + 4096), so that a workload that creeps up
// does not reallocate on every call; the contents are not kept.  The destructor frees it on the current device: aigw_destroy makes
// the context's device current, and waits for its work, before the context's buffers go.
template <class T, bool Pinned = false>
struct Scratch {
  T* p = nullptr;
  size_t cap = 0;   // bytes
  Scratch() = default;
  Scratch(const Scratch&) = delete;
  Scratch& operator=(const Scratch&) = delete;
  ~Scratch() { release(); }
  operator T*() const { return p; }
  cudaError_t ensure(size_t bytes) {
    if (cap >= bytes) return cudaSuccess;
    release();
    const size_t sz = bytes + bytes / 8 + 4096;
    const cudaError_t e = Pinned ? cudaHostAlloc((void**)&p, sz, cudaHostAllocMapped) : cudaMalloc((void**)&p, sz);
    if (e != cudaSuccess) { p = nullptr; return e; }
    cap = sz;
    return cudaSuccess;
  }
  void swap(Scratch& o) { std::swap(p, o.p); std::swap(cap, o.cap); }

 private:
  void release() {
    if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
  }
};
template <class T> using PinnedScratch = Scratch<T, true>;

static constexpr int kSlots = 3;
static bool plain_json_text(const char* s) { for (; *s; s++) { unsigned char c = (unsigned char)*s; if (c < 0x20 || c > 0x7e || c == '"' || c == '\\') return false; } return true; }

struct ChunkSlot {
  Scratch<uint8_t> d_in;
  Scratch<uint64_t> d_off; Scratch<uint32_t> d_len; Scratch<aigw_doc_result> d_res;
  Scratch<uint32_t> d_map;   // size-class bucketing: documents of the chunk grouped by class
  Scratch<uint8_t> d_out;
  cudaEvent_t ev_h2d, ev_k1, ev_done;
};

struct aigw_bpe { Scratch<uint2> d_table; Scratch<uint16_t> d_b2i; uint32_t slots = 0; };

struct aigw_ctx {
  int device = 0, sm_count = 0;
  cudaStream_t s_compute = nullptr, s_h2d = nullptr, s_d2h = nullptr;
  std::string err;
  // counters for the device API (ring so independent launches do not share a counter)
  Scratch<unsigned int> d_counters; int counter_next = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  ChunkSlot slot[kSlots];
  // host-API output (pinned)
  PinnedScratch<uint8_t> h_out;
  PinnedScratch<aigw_doc_result> h_res;
  long small_max = -1;   // aigw_chat_set_small_batch; -1: AIGW_SMALL_MAX or 512
  // large embeddings requests (aigw_embeddings_count_device): token workspace, text table, counts
  Scratch<uint32_t> d_emb_tok; Scratch<uint64_t> d_emb_toff; Scratch<uint32_t> d_emb_tlen; Scratch<uint32_t> d_emb_cnt;
  // large rerank requests (aigw_rerank_translate_large_device): token and depth workspace, splice table
  Scratch<uint32_t> d_rr_tok; Scratch<uint8_t> d_rr_dep; Scratch<RerankSplice> d_rr_splice;
  // large embeddings translations (aigw_embeddings_translate_large_device): one workspace slice per CTA (tokens, escapes, ops, scratch)
  Scratch<uint8_t> d_el_ws;
  // large chat passthroughs (aigw_chat_translate_large_device): one workspace slice per CTA (tokens, jump table, escape counts, arguments)
  Scratch<uint8_t> d_cl_ws;
  // large chat requests to AWS Bedrock (aigw_chat_bedrock_translate_large_device): chat_large's slice, then ops and scratch
  Scratch<uint8_t> d_bl_ws;
  // large chat requests to Anthropic on GCP Vertex AI / AWS Bedrock (aigw_chat_anthropic_translate_large_device), to Gemini on
  // GCP Vertex AI (aigw_chat_gemini_translate_large_device) and large /v1/messages requests to OpenAI / AWS Bedrock Converse
  // (aigw_messages_translate_large_device): the same slice layout.  The three calls share it, as one device call is in flight per
  // context; another grow-only workspace would hold up to 1 GiB more device memory (about 1 GB at 128 KiB bodies).
  Scratch<uint8_t> d_al_ws;
  // large /v1/responses requests (aigw_responses_translate_large_device): one workspace slice per CTA (tokens, jump table, escape counts)
  Scratch<uint8_t> d_rl_ws;
  // large /v1/completions requests (aigw_completions_translate_large_device): tokens, jump table, escape counts, flat-array flags
  Scratch<uint8_t> d_cpl_ws;
  PinnedScratch<uint8_t> h_small;   // small-batch path: tables + bodies, read by the kernel in place
  // chat workspace (intermediates of one sub-batch) + per-stage timing events
  Scratch<uint8_t> d_work;
  Scratch<unsigned long long> d_used_arr; PinnedScratch<unsigned long long> h_used_arr;  // per-chunk bump counters
  cudaEvent_t stage_ev[64]; float stage_ms[3] = {0, 0, 0}; int last_launches = 0;
  bool profile_stages = false;   // aigw_chat_set_profile: next device calls run the stages back to back on one stream and time them
  Scratch<uint8_t> d_stage[6];   // HostStage: one buffer per input table or output area of a single-shot host call (six at most)
  Scratch<uint8_t> d_bs_work;    // bedrock stream workspace (records + counts)
  PinnedScratch<uint8_t> h_chunk_res;   // chunk_pipeline: the mapped result table
  std::vector<uint32_t> h_map;   // size-class bucketing scratch (host)
  // ---- stateful response streams (aigw_stream_*): device-resident slots + per-call staging
  struct StreamPool {
    std::mutex mu;
    Scratch<StreamSlot> d_slots; uint32_t cap = 0;   // cap: slots
    std::vector<uint32_t> free_list, carry, gen, stamp, kind, model_len; std::vector<uint8_t> open; uint32_t call_no = 0;   // kind, model_len: the slot's cfg (stream_out_cap)
    PinnedScratch<uint8_t> h_in; Scratch<uint8_t> d_in;
    PinnedScratch<StreamStep> h_steps; Scratch<StreamStep> d_steps;
    Scratch<aigw_chunk_result> d_res; PinnedScratch<aigw_chunk_result> h_res;
    Scratch<uint8_t> d_out; Scratch<uint8_t> d_packed; PinnedScratch<uint8_t> h_packed;
    Scratch<unsigned long long> d_used; PinnedScratch<unsigned long long> h_used;
    Scratch<uint8_t> d_tmpl; Scratch<uint32_t> d_ids; PinnedScratch<uint32_t> h_ids;
  } sp;
};

// k adjacent counters of the context's ring, zeroed on st
static int take_counters(aigw_ctx* ctx, uint32_t k, cudaStream_t st, unsigned int** out) {
  int at = ctx->counter_next & 255;
  if (at + (int)k > 256) at = 0;
  ctx->counter_next = at + (int)k;
  *out = ctx->d_counters + at;
  CK(cudaMemsetAsync(*out, 0, k * sizeof(unsigned int), st));
  return 0;
}

// launch() on st; when kernel_ms is non-null, also wait for it and store its CUDA-event time there
template <class F>
static int timed(aigw_ctx* ctx, cudaStream_t st, float* kernel_ms, F&& launch) {
  if (kernel_ms) CK(cudaEventRecord(ctx->ev0, st));
  if (int rc = launch()) return rc;
  if (kernel_ms) { CK(cudaEventRecord(ctx->ev1, st)); CK(cudaEventSynchronize(ctx->ev1)); CK(cudaEventElapsedTime(kernel_ms, ctx->ev0, ctx->ev1)); }
  return 0;
}

// Staging of the single-shot host calls: each stages its inputs with in() / span(), takes its output areas with out(), runs its
// *_device form on st, copies its outputs back with back() and ends with wait(): the call's one synchronisation, after which it
// reports the bytes the call copied in and out.  Every table and output area of a call gets a d_stage buffer of its own, in the
// order the call asks for them; no other call uses these buffers.  The first failure is kept in rc: later steps do nothing and
// hand out null pointers, so a call checks rc once before its launch.
struct HostStage {
  aigw_ctx* const ctx;
  const cudaStream_t st;
  int rc = 0, next = 0;
  uint64_t h2d = 0, d2h = 0;   // bytes copied in and out
  explicit HostStage(aigw_ctx* c) : ctx(c), st(c->s_compute) {}

  template <class F> void step(F&& f) { if (!rc) rc = f(); }
  template <class T> T* out(size_t count) {   // 64 bytes of slack: kernels may read a little past a body
    Scratch<uint8_t>& b = ctx->d_stage[next++];
    step([&] { CK(b.ensure(count * sizeof(T) + 64)); return 0; });
    return rc ? nullptr : (T*)b.p;
  }
  template <class T> const T* in(const T* host, size_t count) {
    T* dev = out<T>(count);
    step([&] { CK(cudaMemcpyAsync(dev, host, count * sizeof(T), cudaMemcpyHostToDevice, st)); return 0; });
    h2d += count * sizeof(T);
    return dev;
  }
  // Body i of a (bytes, offsets, lens) table is bytes[offsets[i] .. offsets[i]+lens[i]), in any order.  One copy of the span from the
  // lowest start, rounded down to 16, to the highest end; the device pointer is rebased so that the offsets index it unchanged and
  // every body keeps its alignment modulo 16.
  const uint8_t* span(const uint8_t* bytes, const uint64_t* offsets, const uint32_t* lens, uint32_t n, uint64_t* span_bytes = nullptr) {
    uint64_t lo = ~0ull, hi = 0;
    for (uint32_t i = 0; i < n; i++) { if (offsets[i] < lo) lo = offsets[i]; if (offsets[i] + lens[i] > hi) hi = offsets[i] + lens[i]; }
    lo &= ~15ull;
    if (span_bytes) *span_bytes = hi - lo;
    const uint8_t* dev = in(bytes + lo, hi - lo);
    return rc ? nullptr : dev - lo;
  }
  template <class T> void back(T* host, const T* dev, size_t count) {
    step([&] { CK(cudaMemcpyAsync(host, dev, count * sizeof(T), cudaMemcpyDeviceToHost, st)); return 0; });
    d2h += count * sizeof(T);
  }
  int wait(uint64_t* h2d_bytes = nullptr, uint64_t* d2h_bytes = nullptr) {
    step([&] { CK(cudaStreamSynchronize(st)); return 0; });
    if (!rc && h2d_bytes) *h2d_bytes = h2d;
    if (!rc && d2h_bytes) *d2h_bytes = d2h;
    return rc;
  }
};

// Pipeline chunks of the host calls: chunk c is documents [cb[c], cb[c+1]).  A chunk holds at least one document and ends before
// the first document i with end(i) - start(first document of the chunk) > budget.
template <class S, class E>
static std::vector<uint32_t> chunk_bounds(uint32_t n, uint64_t budget, S&& start, E&& end) {
  std::vector<uint32_t> cb{0};
  uint64_t s = start(0);
  for (uint32_t i = 0; i < n; i++)
    if (end(i) - s > budget && i > cb.back()) { cb.push_back(i); s = start(i); }
  cb.push_back(n);
  return cb;
}

// response direction (AIGW_SCHEMA_RESP_*, any backend): the bodies are upstream responses
static bool response_dir(const aigw_backend_cfg* cfg) { return cfg && (cfg->schema & 48) == AIGW_SCHEMA_RESP_AWS_BEDROCK; }

// the length a body is planned at: response bodies expand (escaped tool arguments, configuration text), so they get a roomier size class
static uint32_t class_len(const aigw_backend_cfg* cfg, uint32_t len) {
  if (!response_dir(cfg)) return len;
  uint64_t m = (uint64_t)len * 4; if (m < 5120) m = 5120; if (m > 65536) m = len > 65536u ? len : 65536u; return (uint32_t)m;
}

// the buffers of one launch (out_bias: where `out` lies in the arena the records' out_off index)
static void chat_buffers(ChatParams& P, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, uint8_t* out, uint64_t out_capacity,
                         aigw_doc_result* results, unsigned long long* out_used, uint64_t out_bias, const uint32_t* doc_map) {
  P.bodies = bodies; P.offsets = offsets; P.lens = lens; P.n = n; P.out = out; P.out_capacity = out_capacity;
  P.results = results; P.out_used = out_used; P.next_doc = nullptr; P.out_bias = out_bias; P.doc_map = doc_map;
}

static void fill_params(ChatParams& P, const aigw_backend_cfg* cfg) {
  P.schema = cfg ? cfg->schema : AIGW_SCHEMA_OPENAI;
  P.cost_configured = cfg ? cfg->cost_configured : 0;
  P.force_mutation = cfg ? cfg->force_body_mutation : 0;
  P.override_len = 0; P.prefix_len = 0; P.version_len = 0; memset(P.api_version, 0, sizeof P.api_version);
  if (cfg && cfg->api_version) { size_t n = strlen(cfg->api_version); if (n > sizeof P.api_version) n = sizeof P.api_version; memcpy(P.api_version, cfg->api_version, n); P.version_len = (uint16_t)n; }
  memset(P.override_model, 0, sizeof P.override_model); memset(P.openai_path, 0, sizeof P.openai_path);
  if (cfg && cfg->model_name_override) {
    size_t n = strlen(cfg->model_name_override); if (n > sizeof P.override_model) n = sizeof P.override_model;
    memcpy(P.override_model, cfg->model_name_override, n); P.override_len = (uint16_t)n;
  }
  // path.Join("/", prefix, "chat/completions") (openai_openai.go:30), "embeddings", "responses" (openai_responses.go:52),
  // "completions" (openai_completions.go:26); rerank below
  std::string pfx = (cfg && cfg->openai_prefix) ? cfg->openai_prefix : "v1";
  while (!pfx.empty() && pfx.front() == '/') pfx.erase(0, 1);
  while (!pfx.empty() && pfx.back() == '/') pfx.pop_back();
  const char* endpoint = !cfg ? "chat/completions" : (cfg->schema & AIGW_SCHEMA_COMPLETIONS) ? "completions" : (cfg->schema & AIGW_SCHEMA_RESPONSES) ? "responses" : (cfg->schema & AIGW_SCHEMA_EMBEDDINGS) ? "embeddings" : "chat/completions";
  std::string path = "/" + (pfx.empty() ? std::string() : pfx + "/") + endpoint;
  if (cfg && (cfg->schema & AIGW_SCHEMA_RERANK)) {
    // path.Join("/", version, "rerank") (cohere_rerank_v2.go:26): the cleaned path, whose "." and ".." segments and doubled slashes
    // are resolved (".." at the root stays at the root).  A path longer than openai_path leaves prefix_len 0 and the walk declines.
    const std::string v = cfg->api_version ? cfg->api_version : "";
    std::vector<std::string> segs;
    for (size_t b = 0; b <= v.size();) {
      size_t e = v.find('/', b); if (e == std::string::npos) e = v.size();
      const std::string s = v.substr(b, e - b);
      if (s == "..") { if (!segs.empty()) segs.pop_back(); }
      else if (!s.empty() && s != ".") segs.push_back(s);
      b = e + 1;
    }
    path.clear();
    for (const std::string& s : segs) path += "/" + s;
    path += "/rerank";
    if (path.size() > sizeof P.openai_path) path.clear();
  }
  if (path.size() > sizeof P.openai_path) path.resize(sizeof P.openai_path);
  memcpy(P.openai_path, path.data(), path.size()); P.prefix_len = (uint16_t)path.size();
  P.created = 0; P.rid_len = 0; memset(P.response_id, 0, sizeof P.response_id);
  if (response_dir(cfg)) {
    P.created = cfg->created;
    if (cfg->response_id) { size_t n = strlen(cfg->response_id); if (n > sizeof P.response_id) n = sizeof P.response_id; memcpy(P.response_id, cfg->response_id, n); P.rid_len = (uint16_t)n; }
  }
}

namespace aigw {
int ctx_device(const aigw_ctx* ctx) { return ctx->device; }
bool chat_small_fits(const aigw_backend_cfg* cfg, uint32_t len) { return len > 0 && class_len(cfg, len) <= kSmallMaxLen; }
cudaError_t chat_small_launch(const aigw_backend_cfg* cfg, const uint8_t* in, const uint64_t* offsets, const uint32_t* lens, const uint64_t* out_slot, uint32_t n, uint8_t* out,
                              aigw_doc_result* results, cudaStream_t st) {
  ChatParams P; fill_params(P, cfg);
  chat_buffers(P, in, offsets, lens, n, out, 0, results, nullptr, 0, nullptr);
  return launch_chat_small(P, 0, n, out_slot, st);
}
}  // namespace aigw

// host loops over the calls of one window (byte staging, result hand-back) run on a few threads when the window is large
template <class F>
static void host_parallel_for(uint32_t n, F&& f) {
  static const unsigned hw = [] { unsigned h = 2; const char* e = getenv("AIGW_HOST_THREADS"); if (e) h = (unsigned)atoi(e); return h < 1 ? 1u : (h > 8 ? 8u : h); }();   // more staging threads slow the DMA that follows
  if (n < 16384 || hw == 1) { f(0u, n); return; }
  std::vector<std::thread> th;
  const uint32_t per = (n + hw - 1) / hw;
  for (unsigned t = 1; t < hw; t++) { const uint32_t b = t * per, e = b + per < n ? b + per : n; if (b < e) th.emplace_back([&f, b, e] { f(b, e); }); }
  f(0u, per < n ? per : n);
  for (auto& x : th) x.join();
}

// One chunk of chunk_pipeline: items [first, first + n) of the call, staged in a slot.
template <class R>
struct PipeChunk {
  uint32_t first, n;
  const uint8_t* bytes;            // the staged input, indexed by the caller's offsets
  const uint64_t* off;             // the staged offset table from item `first` on: n + 1 entries, or n with a length table
  const uint32_t* len;             // the staged length table, or null
  uint8_t* out; uint64_t out_cap;  // the chunk's part of the output arena (device view)
  uint64_t out_bias;               // where that part starts in the arena: added to the records' out_off
  unsigned long long* out_used;    // the chunk's bump counter, zeroed
  R* results;                      // results of the chunk's items (device view)
  uint64_t max_in; uint32_t max_n; // the largest chunk of the call: sizes a workspace the chunks share
};

// The host-buffer pipeline of aigw_bedrock_stream_host and aigw_body_mutate_host.  Item i is bytes[off[i] .. off[i+1]) (len null:
// an n+1 offset table) or bytes[off[i] .. off[i]+len[i]) (bodies in arena order).  The items are cut into chunks of about `budget`
// bytes that alternate between two slots: the H2D copy of chunk c+1 (s_h2d) overlaps the kernels of chunk c (s_compute), which
// store the records and results straight into mapped pinned host memory; one synchronisation at the end.  out_cap(in_bytes, items)
// is a chunk's output capacity; launch(chunk) starts `launches` kernels on s_compute.
template <class Out, class Cap, class Launch>
static int chunk_pipeline(aigw_ctx* ctx, const uint8_t* bytes, const uint64_t* off, const uint32_t* len, uint32_t n, uint64_t budget,
                          Cap&& out_cap_of, uint32_t launches, Launch&& launch, Out* out) {
  using R = std::remove_const_t<std::remove_pointer_t<decltype(out->results)>>;
  auto end = [&](uint32_t i) { return len ? off[i] + len[i] : off[i + 1]; };
  const std::vector<uint32_t> cb = chunk_bounds(n, budget, [&](uint32_t i) { return off[i]; }, end);
  const int nch = (int)cb.size() - 1;
  std::vector<uint64_t> in_bytes(nch), out_cap(nch), out_base(nch);
  uint64_t max_in = 0, total_cap = 0; uint32_t max_n = 0;
  for (int c = 0; c < nch; c++) {
    const uint32_t b = cb[c], nd = cb[c + 1] - b;
    in_bytes[c] = end(cb[c + 1] - 1) - off[b];
    if (in_bytes[c] > max_in) max_in = in_bytes[c]; if (nd > max_n) max_n = nd;
    out_cap[c] = out_cap_of(in_bytes[c], nd);
    out_base[c] = total_cap; total_cap += out_cap[c];
  }
  const int nslots = nch < 2 ? 1 : 2;
  for (int k = 0; k < nslots; k++) {
    ChunkSlot& S = ctx->slot[k];
    CK(S.d_in.ensure(max_in + 64));
    CK(S.d_off.ensure(((size_t)max_n + 1) * 8));
    if (len) CK(S.d_len.ensure((size_t)max_n * 4));
  }
  CK(ctx->h_out.ensure(total_cap));
  CK(ctx->h_chunk_res.ensure((size_t)n * sizeof(R)));
  CK(ctx->d_used_arr.ensure((size_t)nch * 8)); CK(ctx->h_used_arr.ensure((size_t)nch * 8));
  uint8_t* dev_out = nullptr; R* dev_res = nullptr;
  CK(cudaHostGetDevicePointer((void**)&dev_out, ctx->h_out, 0));
  CK(cudaHostGetDevicePointer((void**)&dev_res, ctx->h_chunk_res, 0));
  uint64_t h2d = 0;
  CK(cudaMemsetAsync(ctx->d_used_arr, 0, (size_t)nch * 8, ctx->s_compute));
  CK(cudaEventRecord(ctx->ev0, ctx->s_compute));
  for (int c = 0; c < nch; c++) {
    ChunkSlot& S = ctx->slot[c % nslots];
    const uint32_t b = cb[c], nd = cb[c + 1] - b;
    const size_t n_off = len ? nd : (size_t)nd + 1;
    if (c >= nslots) CK(cudaStreamWaitEvent(ctx->s_h2d, S.ev_k1, 0));   // the slot's input has been consumed
    CK(cudaMemcpyAsync(S.d_in, bytes + off[b], in_bytes[c], cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(S.d_off, off + b, n_off * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    if (len) CK(cudaMemcpyAsync(S.d_len, len + b, (size_t)nd * 4, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaEventRecord(S.ev_h2d, ctx->s_h2d));
    h2d += in_bytes[c] + n_off * 8 + (len ? (uint64_t)nd * 4 : 0);
    CK(cudaStreamWaitEvent(ctx->s_compute, S.ev_h2d, 0));
    if (int rc = launch(PipeChunk<R>{b, nd, S.d_in - off[b], S.d_off, len ? (const uint32_t*)S.d_len : nullptr, dev_out + out_base[c], out_cap[c], out_base[c],
                                     ctx->d_used_arr + c, dev_res + b, max_in, max_n}))
      return rc;
    CK(cudaEventRecord(S.ev_k1, ctx->s_compute));
    out->gpu_launches += launches;
  }
  CK(cudaEventRecord(ctx->ev1, ctx->s_compute));
  CK(cudaMemcpyAsync(ctx->h_used_arr, ctx->d_used_arr, (size_t)nch * 8, cudaMemcpyDeviceToHost, ctx->s_compute));
  CK(cudaStreamSynchronize(ctx->s_compute));
  uint64_t d2h = (uint64_t)n * sizeof(R) + (uint64_t)nch * 8;
  for (int c = 0; c < nch; c++) d2h += ctx->h_used_arr[c] < out_cap[c] ? ctx->h_used_arr[c] : out_cap[c];
  float ms = 0; cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1);
  out->results = (const R*)ctx->h_chunk_res.p; out->out = ctx->h_out; out->out_used = total_cap; out->h2d_bytes = h2d; out->d2h_bytes = d2h; out->kernel_ms = ms;
  return 0;
}

extern "C" {

const char* aigw_version(void) { return "aigw_b200 0.1 (sm_90a)"; }

int aigw_init(int device, aigw_ctx** out) {
  *out = nullptr;
  aigw_ctx* ctx = new aigw_ctx();
  ctx->device = device;
  cudaError_t e = cudaSetDevice(device);
  // a failed runtime call leaves its code as the thread's "last error": clear it, or the next launch check of ANOTHER context on this
  // thread (cudaGetLastError after a kernel launch) reports it as its own (found by tests/test_multi_context_gpu.py)
  if (e != cudaSuccess) { fprintf(stderr, "aigw_init: cudaSetDevice(%d): %s\n", device, cudaGetErrorString(e)); (void)cudaGetLastError(); delete ctx; return (int)e; }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) { (void)cudaGetLastError(); delete ctx; return (int)e; }
  ctx->sm_count = prop.multiProcessorCount;
  // sm_90a code runs on compute capability 9.0 and nothing else (architecture-specific features are not forward compatible)
  if (prop.major != 9 || prop.minor != 0) { fprintf(stderr, "aigw_init: device %d is sm_%d%d; this library is built for sm_90a (H100) only\n", device, prop.major, prop.minor); delete ctx; return (int)cudaErrorNoKernelImageForDevice; }
  // every allocation is checked on its own: a half-built context is destroyed, never returned
  auto fail = [&](const char* what, cudaError_t err) { fprintf(stderr, "aigw_init: %s: %s\n", what, cudaGetErrorString(err)); aigw_destroy(ctx); return (int)err; };
#define INIT_CK(x) do { cudaError_t _e = (x); if (_e != cudaSuccess) return fail(#x, _e); } while (0)
  INIT_CK(cudaStreamCreateWithFlags(&ctx->s_compute, cudaStreamNonBlocking));
  INIT_CK(cudaStreamCreateWithFlags(&ctx->s_h2d, cudaStreamNonBlocking));
  INIT_CK(cudaStreamCreateWithFlags(&ctx->s_d2h, cudaStreamNonBlocking));
  INIT_CK(ctx->d_counters.ensure(256 * sizeof(unsigned int)));
  INIT_CK(cudaEventCreate(&ctx->ev0)); INIT_CK(cudaEventCreate(&ctx->ev1));
  for (auto& e2 : ctx->stage_ev) INIT_CK(cudaEventCreate(&e2));
  for (auto& s : ctx->slot) {
    INIT_CK(cudaEventCreateWithFlags(&s.ev_h2d, cudaEventDisableTiming)); INIT_CK(cudaEventCreate(&s.ev_k1)); INIT_CK(cudaEventCreateWithFlags(&s.ev_done, cudaEventDisableTiming));
  }
#undef INIT_CK
  *out = ctx;
  return 0;
}

void aigw_destroy(aigw_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto& s : ctx->slot) {
    cudaEventDestroy(s.ev_h2d); cudaEventDestroy(s.ev_k1); cudaEventDestroy(s.ev_done);
  }
  for (auto& e2 : ctx->stage_ev) cudaEventDestroy(e2);
  cudaEventDestroy(ctx->ev0); cudaEventDestroy(ctx->ev1);
  cudaStreamDestroy(ctx->s_compute); cudaStreamDestroy(ctx->s_h2d); cudaStreamDestroy(ctx->s_d2h);
  delete ctx;
}

// Bind the calling thread (and the threads it starts later) to the CPUs of the NUMA node the GPU hangs off, so that pinned
// arenas allocated afterwards are node-local (first touch) and the copy engines do not cross the socket interconnect
// (VERDICT r1: 8 ranks on one host lost 4x end to end with unbound ranks).  Returns the node, or -1 when it cannot be determined.
int aigw_bind_numa(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) return -1;
  for (char* c = bus; *c; c++) if (*c >= 'A' && *c <= 'F') *c = (char)(*c - 'A' + 'a');
  char path[128]; snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE* f = fopen(path, "r"); if (!f) return -1;
  int node = -1; if (fscanf(f, "%d", &node) != 1) node = -1; fclose(f);
  if (node < 0) return -1;
  snprintf(path, sizeof path, "/sys/devices/system/node/node%d/cpulist", node);
  f = fopen(path, "r"); if (!f) return -1;
  char list[4096] = {0}; if (!fgets(list, sizeof list, f)) { fclose(f); return -1; } fclose(f);
  cpu_set_t want; CPU_ZERO(&want);
  for (char* p = list; *p;) {
    char* end; long a = strtol(p, &end, 10); if (end == p) break; long b = a;
    if (*end == '-') { p = end + 1; b = strtol(p, &end, 10); }
    for (long c = a; c <= b && c < CPU_SETSIZE; c++) CPU_SET((int)c, &want);
    p = *end == ',' ? end + 1 : end; if (*end != ',' ) break;
  }
  cpu_set_t cur; CPU_ZERO(&cur);
  if (sched_getaffinity(0, sizeof cur, &cur) == 0) { cpu_set_t both; CPU_AND(&both, &cur, &want); if (CPU_COUNT(&both) > 0) want = both; }
  if (CPU_COUNT(&want) == 0 || sched_setaffinity(0, sizeof want, &want) != 0) return -1;
  return node;
}

const char* aigw_last_error(aigw_ctx* ctx) { return ctx ? ctx->err.c_str() : "no context"; }
int aigw_device_sm_count(aigw_ctx* ctx) { return ctx->sm_count; }

void* aigw_host_alloc(aigw_ctx* ctx, size_t bytes) { void* p = nullptr; cudaSetDevice(ctx->device); if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { ctx->err = "cudaHostAlloc failed"; return nullptr; } return p; }
void aigw_host_free(aigw_ctx*, void* p) { cudaFreeHost(p); }
void* aigw_device_alloc(aigw_ctx* ctx, size_t bytes) { void* p = nullptr; cudaSetDevice(ctx->device); if (cudaMalloc(&p, bytes) != cudaSuccess) { ctx->err = "cudaMalloc failed"; return nullptr; } return p; }
void aigw_device_free(aigw_ctx* ctx, void* p) { cudaSetDevice(ctx->device); cudaFree(p); }
int aigw_memcpy_h2d(aigw_ctx* ctx, void* dst, const void* src, size_t bytes) { ENTER(); CK(cudaMemcpy(dst, src, bytes, cudaMemcpyHostToDevice)); return 0; }
int aigw_memcpy_d2h(aigw_ctx* ctx, void* dst, const void* src, size_t bytes) { ENTER(); CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost)); return 0; }
int aigw_memset_d(aigw_ctx* ctx, void* dst, int v, size_t bytes) { ENTER(); CK(cudaMemset(dst, v, bytes)); return 0; }
int aigw_sync(aigw_ctx* ctx) { ENTER(); CK(cudaDeviceSynchronize()); return 0; }

// the translate workspace for `docs` documents planned at max_len bytes: two sub-batch slots for a call the paired schedule
// runs, one sub-batch otherwise, at most 3 GiB: the launcher walks a size class in sub-batches that fit it
static int ensure_chat_work(aigw_ctx* ctx, uint32_t max_len, uint32_t docs) {
  size_t need = chat_work_bytes_for(max_len, docs);
  const size_t cap = (size_t)3 << 30, floor1 = chat_work_bytes(max_len, 1024);
  if (need > cap) need = cap > floor1 ? cap : floor1;
  CK(ctx->d_work.ensure(need));
  return 0;
}

static int chat_translate_device_impl(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                      const uint32_t* d_lens, const uint32_t* d_doc_map, uint32_t first, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                      aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams P;
  fill_params(P, cfg);
  chat_buffers(P, d_bodies, d_offsets, d_lens, n, d_out, out_capacity, d_results, (unsigned long long*)d_out_used, 0, d_doc_map);
  const uint32_t ml = class_len(cfg, max_len ? max_len : 65536u);
  const bool stages = ctx->profile_stages && kernel_ms;
  if (int rc = ensure_chat_work(ctx, ml, n)) return rc;
  if (int rc = timed(ctx, st, kernel_ms, [&] {
        CK(launch_chat_translate(P, ml, ctx->device, ctx->sm_count, st, ctx->d_work, ctx->d_work.cap, &ctx->last_launches, stages ? ctx->stage_ev : nullptr, 64, first));
        return 0;
      }))
    return rc;
  if (stages) {
    ctx->stage_ms[0] = ctx->stage_ms[1] = ctx->stage_ms[2] = 0;
    const int nsb = ctx->last_launches / 4;
    for (int sb = 0; sb < nsb && 4 * sb + 3 < 64; sb++) for (int k = 0; k < 3; k++) { float ms = 0; cudaEventElapsedTime(&ms, ctx->stage_ev[4 * sb + k], ctx->stage_ev[4 * sb + k + 1]); ctx->stage_ms[k] += ms; }
  }
  return 0;
}

int aigw_chat_translate_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                               const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                               aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  return chat_translate_device_impl(ctx, cfg, d_bodies, d_offsets, d_lens, nullptr, 0, n, max_len, d_out, out_capacity, d_results, d_out_used, stream, kernel_ms);
}
int aigw_chat_translate_device_mapped(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens,
                                      const uint32_t* d_doc_map, uint32_t first, uint32_t count, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                      aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  return chat_translate_device_impl(ctx, cfg, d_bodies, d_offsets, d_lens, d_doc_map, first, count, max_len, d_out, out_capacity, d_results, d_out_used, stream, kernel_ms);
}

int aigw_chat_set_profile(aigw_ctx* ctx, int on) { ctx->profile_stages = on != 0; return 0; }

/* per-stage CUDA-event times (index, walk, emit) of the last profiled call and the launch count of the last device call */
int aigw_chat_last_profile(aigw_ctx* ctx, float stage_ms[3], int* launches) {
  for (int k = 0; k < 3; k++) stage_ms[k] = ctx->stage_ms[k];
  if (launches) *launches = ctx->last_launches;
  return 0;
}

// Small batches (a single request, or what a batching window collects): one fused kernel, no workspace, no device copies.
// Every body owns a fixed output slot of 3 x its length + 1 KiB (the embeddings -> Vertex instances translation expands short
// inputs up to 5x; a record that does not fit is DECLINED with AIGW_R_ARENA_FULL, never truncated).
// The bodies are packed into a mapped pinned buffer the kernel reads in place, the records and results are stored straight
// into the pinned output arenas, and the call is launch + kernel + one synchronisation.
static int chat_small_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  uint64_t in_bytes = 0, out_bytes = 0;
  for (uint32_t i = 0; i < n; i++) { in_bytes += (((uint64_t)lens[i] + 15u) & ~15ull) + 16; out_bytes += ((uint64_t)lens[i] * 3 + 1024 + 15) & ~15ull; }
  const size_t tab = (((size_t)n + 1) * 16 + (size_t)n * 4 + 63) & ~(size_t)63;
  CK(ctx->h_small.ensure(tab + in_bytes + 64));
  CK(ctx->h_out.ensure(out_bytes + 64));
  CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result)));
  uint64_t* h_off = (uint64_t*)ctx->h_small.p; uint64_t* h_slot = h_off + n + 1; uint32_t* h_len = (uint32_t*)(h_slot + n + 1);
  uint8_t* h_in = ctx->h_small + tab;
  uint64_t o = 0, so = 0;
  for (uint32_t i = 0; i < n; i++) {
    h_off[i] = o; h_slot[i] = so; h_len[i] = lens[i];
    memcpy(h_in + o, bodies + offsets[i], lens[i]);
    o += (((uint64_t)lens[i] + 15u) & ~15ull) + 16; so += ((uint64_t)lens[i] * 3 + 1024 + 15) & ~15ull;
  }
  h_off[n] = o; h_slot[n] = so;
  uint8_t* d_small = nullptr; uint8_t* d_out = nullptr; aigw_doc_result* d_res = nullptr;
  CK(cudaHostGetDevicePointer((void**)&d_small, ctx->h_small, 0)); CK(cudaHostGetDevicePointer((void**)&d_out, ctx->h_out, 0)); CK(cudaHostGetDevicePointer((void**)&d_res, ctx->h_res, 0));
  ChatParams P; fill_params(P, cfg);
  chat_buffers(P, d_small + tab, (const uint64_t*)d_small, (const uint32_t*)(d_small + ((size_t)n + 1) * 16), n, d_out, so, d_res, nullptr, 0, nullptr);
  static const bool dbg = getenv("AIGW_SMALL_DBG") != nullptr;
  static unsigned int* h_dbg = nullptr;
  if (dbg) { if (!h_dbg) cudaHostAlloc((void**)&h_dbg, 64, cudaHostAllocDefault); P.next_doc = h_dbg; }
  CK(cudaEventRecord(ctx->ev0, ctx->s_compute));
  CK(launch_chat_small(P, 0, n, (const uint64_t*)d_small + n + 1, ctx->s_compute));
  CK(cudaEventRecord(ctx->ev1, ctx->s_compute));
  CK(cudaEventSynchronize(ctx->ev1));
  float kms = 0; cudaEventElapsedTime(&kms, ctx->ev0, ctx->ev1);
  if (dbg) fprintf(stderr, "small n=%u kernel %.1f us  clocks: load %u index %u walk %u emit %u\n", n, kms * 1e3f, h_dbg[0], h_dbg[1], h_dbg[2], h_dbg[3]);
  uint64_t produced = 0;
  for (uint32_t i = 0; i < n; i++) if (ctx->h_res[i].status == AIGW_OK) produced += ((uint64_t)ctx->h_res[i].path_len + ctx->h_res[i].body_len + 15u) & ~15ull;
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = so; out->h2d_bytes = in_bytes + tab; out->d2h_bytes = produced + (uint64_t)n * sizeof(aigw_doc_result);
  out->gpu_launches = 1; out->kernel_ms = kms;
  return 0;
}

void aigw_chat_set_small_batch(aigw_ctx* ctx, int max_docs) { if (ctx) ctx->small_max = max_docs; }

int aigw_chat_translate_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                             const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  // Three-stage pipeline over 256 MiB chunks, both PCIe directions busy at once:
  //   copy engine A   H2D of chunk c+1                               (s_h2d)
  //   SMs             index / sort / walk / emit of chunk c → device (s_compute)
  //   copy engine B   D2H of chunk c-1: exactly the bytes the emit stage produced + the chunk's result table (s_d2h)
  // The host runs one chunk behind the GPU (it waits for chunk c-1's byte count while chunk c's kernels are queued).
  memset(out, 0, sizeof *out);
  if (n == 0) return 0;
  ENTER();
  {
    static const long env_small_max = getenv("AIGW_SMALL_MAX") ? atol(getenv("AIGW_SMALL_MAX")) : 512;   // 0 disables the fused small-batch path
    if ((long)n <= (ctx->small_max >= 0 ? ctx->small_max : env_small_max)) {
      uint32_t ml = 0; for (uint32_t i = 0; i < n; i++) if (lens[i] > ml) ml = lens[i];
      if (class_len(cfg, ml) <= kSmallMaxLen) return chat_small_host(ctx, cfg, bodies, offsets, lens, n, out);
    }
  }
  static const uint64_t kChunkBytes = (uint64_t)(getenv("AIGW_CHUNK_MB") ? atol(getenv("AIGW_CHUNK_MB")) : 256) << 20;   // pipeline granularity (fill / drain cost vs per-chunk launches)
  const std::vector<uint32_t> cb = chunk_bounds(n, kChunkBytes, [&](uint32_t i) { return offsets[i]; }, [&](uint32_t i) { return offsets[i] + (((uint64_t)lens[i] + 15u) & ~15ull); });
  uint32_t max_len = 0;
  for (uint32_t i = 0; i < n; i++) if (lens[i] > max_len) max_len = lens[i];
  const int nch = (int)cb.size() - 1;
  uint64_t max_in = 0, max_out = 0; uint32_t max_docs = 0;
  std::vector<uint64_t> in_bytes(nch), out_cap(nch), out_base(nch);
  uint64_t total_out_cap = 0;
  for (int c = 0; c < nch; c++) {
    const uint32_t b = cb[c], e = cb[c + 1];
    const uint64_t ib = offsets[e - 1] + (((uint64_t)lens[e - 1] + 15u) & ~15ull) - offsets[b] + 16;
    in_bytes[c] = ib; if (ib > max_in) max_in = ib; if (e - b > max_docs) max_docs = e - b;
    out_cap[c] = ((ib + ib / 4 + (uint64_t)(e - b) * 528 + 255) & ~255ull);
    if (out_cap[c] > max_out) max_out = out_cap[c];
    out_base[c] = total_out_cap; total_out_cap += out_cap[c];
  }
  const int nslots = nch < kSlots ? nch : kSlots;
  for (int s = 0; s < nslots; s++) {
    ChunkSlot& S = ctx->slot[s];
    CK(S.d_in.ensure(max_in + 64));
    CK(S.d_out.ensure(max_out + 64));
    CK(S.d_off.ensure((size_t)max_docs * 8)); CK(S.d_len.ensure((size_t)max_docs * 4)); CK(S.d_res.ensure((size_t)max_docs * sizeof(aigw_doc_result)));
  }
  max_len = class_len(cfg, max_len);
  // size classes (the kernels' shared-memory footprints, chat_kernel.cu launch_chat_translate)
  static const uint32_t kClsMax[6] = {2048, 5120, 9216, 17408, 33792, 65536};
  auto cls_of = [&](uint32_t len) { const uint32_t l = class_len(cfg, len); int k = 0; while (k < 5 && l > kClsMax[k]) k++; return k; };
  if (int rc = ensure_chat_work(ctx, max_len, max_docs)) return rc;
  CK(ctx->h_out.ensure(total_out_cap));
  CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result)));
  CK(ctx->d_used_arr.ensure((size_t)nch * 8)); CK(ctx->h_used_arr.ensure((size_t)nch * 8));

  ChatParams P0; fill_params(P0, cfg);
  uint64_t h2d = 0, d2h = (uint64_t)n * sizeof(aigw_doc_result) + (uint64_t)nch * 8;
  CK(cudaMemsetAsync(ctx->d_used_arr, 0, (size_t)nch * 8, ctx->s_compute));
  CK(cudaEventRecord(ctx->ev0, ctx->s_compute));
  auto drain = [&](int k) -> int {   // chunk k's kernels are done: move exactly what they produced
    ChunkSlot& S = ctx->slot[k % nslots];
    CK(cudaEventSynchronize(S.ev_k1));
    const uint64_t used = ctx->h_used_arr[k] < out_cap[k] ? ctx->h_used_arr[k] : out_cap[k];
    d2h += used;
    const uint32_t b = cb[k], nd = cb[k + 1] - b;
    if (used) CK(cudaMemcpyAsync(ctx->h_out + out_base[k], S.d_out, used, cudaMemcpyDeviceToHost, ctx->s_d2h));
    CK(cudaMemcpyAsync(ctx->h_res + b, S.d_res, (size_t)nd * sizeof(aigw_doc_result), cudaMemcpyDeviceToHost, ctx->s_d2h));
    CK(cudaEventRecord(S.ev_done, ctx->s_d2h));
    return 0;
  };
  for (int c = 0; c < nch; c++) {
    ChunkSlot& S = ctx->slot[c % nslots];
    const uint32_t b = cb[c], e = cb[c + 1], nd = e - b;
    if (c >= nslots) {
      CK(cudaStreamWaitEvent(ctx->s_h2d, S.ev_k1, 0));                       // the slot's input has been consumed
      CK(cudaStreamWaitEvent(ctx->s_compute, S.ev_done, 0));                 // the slot's output has left the device
    }
    CK(cudaMemcpyAsync(S.d_in, bodies + offsets[b], in_bytes[c] - 16, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(S.d_off, offsets + b, (size_t)nd * 8, cudaMemcpyHostToDevice, ctx->s_h2d));
    CK(cudaMemcpyAsync(S.d_len, lens + b, (size_t)nd * 4, cudaMemcpyHostToDevice, ctx->s_h2d));
    // size-class bucketing: a chunk whose documents span several classes is launched class by class over a document map,
    // so that a few large bodies do not force the small ones into the large class's shared-memory footprint
    uint32_t cls_cnt[6] = {0, 0, 0, 0, 0, 0};
    for (uint32_t i = b; i < e; i++) cls_cnt[cls_of(lens[i])]++;
    int n_cls = 0, top_cls = 0; for (int k = 0; k < 6; k++) if (cls_cnt[k]) { n_cls++; top_cls = k; }
    static const bool no_bucketing = getenv("AIGW_NO_BUCKETING") != nullptr;   // A/B switch for the Zipf bench
    if (no_bucketing) n_cls = 1;
    uint32_t cls_start[7] = {0, 0, 0, 0, 0, 0, 0};
    if (n_cls > 1) {
      for (int k = 0; k < 6; k++) cls_start[k + 1] = cls_start[k] + cls_cnt[k];
      ctx->h_map.resize(nd);
      uint32_t cur[6]; for (int k = 0; k < 6; k++) cur[k] = cls_start[k];
      for (uint32_t i = b; i < e; i++) ctx->h_map[cur[cls_of(lens[i])]++] = i;
      CK(S.d_map.ensure((size_t)nd * 4));
      CK(cudaMemcpyAsync(S.d_map, ctx->h_map.data(), (size_t)nd * 4, cudaMemcpyHostToDevice, ctx->s_h2d));   // pageable source: staged before the call returns
      h2d += (uint64_t)nd * 4;
    }
    CK(cudaEventRecord(S.ev_h2d, ctx->s_h2d));
    h2d += in_bytes[c] - 16 + (uint64_t)nd * 12;
    CK(cudaStreamWaitEvent(ctx->s_compute, S.ev_h2d, 0));
    // documents keep their global index: kernels address offsets/lens/results with doc0 + i (or doc_map[i]), and the absolute
    // offsets index straight into the chunk
    ChatParams P = P0;
    chat_buffers(P, S.d_in - offsets[b], S.d_off - b, S.d_len - b, nd, S.d_out, out_cap[c], S.d_res - b, ctx->d_used_arr + c, out_base[c],
                 n_cls > 1 ? (const uint32_t*)S.d_map : nullptr);
    if (n_cls <= 1) {
      int nl = 0;
      CK(launch_chat_translate(P, kClsMax[top_cls], ctx->device, ctx->sm_count, ctx->s_compute, ctx->d_work, ctx->d_work.cap, &nl, nullptr, 0, b));
      out->gpu_launches += nl;
    } else {
      for (int k = 0; k < 6; k++) {
        if (!cls_cnt[k]) continue;
        int nl = 0;
        P.n = cls_cnt[k];
        CK(launch_chat_translate(P, kClsMax[k], ctx->device, ctx->sm_count, ctx->s_compute, ctx->d_work, ctx->d_work.cap, &nl, nullptr, 0, cls_start[k]));
        out->gpu_launches += nl;
      }
    }
    CK(cudaMemcpyAsync(ctx->h_used_arr + c, ctx->d_used_arr + c, 8, cudaMemcpyDeviceToHost, ctx->s_compute));
    CK(cudaEventRecord(S.ev_k1, ctx->s_compute));
    if (c >= 1) { const int rc = drain(c - 1); if (rc) return rc; }
  }
  CK(cudaEventRecord(ctx->ev1, ctx->s_compute));
  { const int rc = drain(nch - 1); if (rc) return rc; }
  CK(cudaStreamSynchronize(ctx->s_d2h));
  CK(cudaStreamSynchronize(ctx->s_compute));
  float ms_total = 0; cudaEventElapsedTime(&ms_total, ctx->ev0, ctx->ev1);
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = total_out_cap; out->h2d_bytes = h2d; out->d2h_bytes = d2h; out->kernel_ms = ms_total;
  return 0;
}

// ------------------------------------------------------------------ K4: BPE token count
int aigw_bpe_load(aigw_ctx* ctx, const uint16_t* byte_to_id, const uint32_t* merges, uint32_t n_merges, aigw_bpe** out) {
  if (!ctx || !byte_to_id || (!merges && n_merges) || !out || n_merges >= 65535u) return -2;
  // ids stop at 65534: the pair (65535, 65535) would have key 0xFFFFFFFF, the empty-slot marker of the table
  for (uint32_t i = 0; i < 256; i++) if (byte_to_id[i] >= 65535u) return -2;
  for (uint32_t r = 0; r < n_merges * 3; r++) if (merges[r] >= 65535u) return -2;
  ENTER();
  uint32_t slots = 1024; while (slots < n_merges * 2u) slots <<= 1;
  if (bpe_smem_bytes(slots) > 220u * 1024u) { ctx->err = "aigw_bpe_load: merge table does not fit shared memory"; return -2; }
  std::vector<uint2> tab(slots, make_uint2(0xffffffffu, 0xffffffffu));
  for (uint32_t r = 0; r < n_merges; r++) {
    const uint32_t key = (merges[3 * r] << 16) | merges[3 * r + 1];
    uint32_t h = key * 0x9E3779B1u; h ^= h >> 15;
    uint32_t s = h & (slots - 1);
    bool dup = false;
    while (tab[s].x != 0xffffffffu) { if (tab[s].x == key) { dup = true; break; } s = (s + 1) & (slots - 1); }
    if (dup) continue;   // the first rank of a pair wins (a well-formed merge list has no duplicates)
    tab[s] = make_uint2(key, (r << 16) | merges[3 * r + 2]);
  }
  std::unique_ptr<aigw_bpe> b(new aigw_bpe());   // freed with its buffers unless it is handed out
  b->slots = slots;
  CK(b->d_table.ensure((size_t)slots * 8)); CK(b->d_b2i.ensure(512));
  CK(cudaMemcpy(b->d_table, tab.data(), (size_t)slots * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(b->d_b2i, byte_to_id, 512, cudaMemcpyHostToDevice));
  *out = b.release();
  return 0;
}
void aigw_bpe_free(aigw_ctx* ctx, aigw_bpe* b) { if (!b) return; if (ctx) cudaSetDevice(ctx->device); delete b; }

int aigw_bpe_count_device(aigw_ctx* ctx, const aigw_bpe* bpe, const uint8_t* d_text, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n, uint32_t* d_counts,
                          void* stream, float* kernel_ms) {
  if (!ctx || !bpe) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  BpeParams P; P.text = d_text; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.counts = d_counts; P.table = bpe->d_table; P.slots = bpe->slots; P.byte_to_id = bpe->d_b2i;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_bpe_count(P, ctx->sm_count, st)); return 0; });
}

int aigw_bpe_count_host(aigw_ctx* ctx, const aigw_bpe* bpe, const uint8_t* text, const uint64_t* offsets, const uint32_t* lens, uint32_t n, uint32_t* counts,
                        uint64_t* h2d_bytes, uint64_t* d2h_bytes, float* kernel_ms) {
  if (!ctx || !bpe) return -2;
  if (n == 0) return 0;
  ENTER();
  HostStage S(ctx);
  const uint8_t* d_text = S.span(text, offsets, lens, n);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  uint32_t* d_counts = S.out<uint32_t>(n);
  if (S.rc) return S.rc;
  if (int rc = aigw_bpe_count_device(ctx, bpe, d_text, d_off, d_len, n, d_counts, S.st, kernel_ms)) return rc;
  S.back(counts, d_counts, n);
  return S.wait(h2d_bytes, d2h_bytes);
}

// ------------------------------------------------------------------ large /v1/embeddings requests: ParseBody + BPE count (BASELINE config 3)
int aigw_embeddings_count_device(aigw_ctx* ctx, const aigw_bpe* bpe, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n, uint32_t max_len,
                                 uint64_t total_bytes, aigw_emb_count_result* d_results, void* stream, float* kernel_ms) {
  if (!ctx || !bpe) return -2;
  if (kernel_ms) kernel_ms[0] = kernel_ms[1] = kernel_ms[2] = kernel_ms[3] = 0;
  if (n == 0) return 0;
  ENTER_ON(stream);
  // every input costs at least three request bytes (two quotes and a comma); one row per four bytes covers inputs of two characters and up,
  // a request that would overflow the table is declined (AIGW_R_ARENA_FULL)
  const uint64_t text_cap64 = total_bytes / 4 + 1024;
  if (text_cap64 >= (1ull << 32)) { ctx->err = "aigw_embeddings_count: more than 16 GiB in one call; split it into waves"; return -2; }
  const uint32_t text_cap = (uint32_t)text_cap64;
  const uint32_t tok_cap = max_len / 2 + 64;
  const int grid = emb_scan_grid(ctx->sm_count);
  CK(ctx->d_emb_tok.ensure((size_t)grid * tok_cap * 4));
  CK(ctx->d_emb_toff.ensure((size_t)text_cap * 8));
  CK(ctx->d_emb_tlen.ensure((size_t)text_cap * 4));
  CK(ctx->d_emb_cnt.ensure((size_t)text_cap * 4));
  unsigned int* c0;
  if (int rc = take_counters(ctx, 3, st, &c0)) return rc;
  unsigned int* c1 = c0 + 1; unsigned int* c2 = c0 + 2;
  EmbScanParams E; E.bodies = d_bodies; E.offsets = d_offsets; E.lens = d_lens; E.n = n; E.results = d_results; E.tok_ws = ctx->d_emb_tok; E.tok_cap = tok_cap;
  E.text_off = ctx->d_emb_toff; E.text_len = ctx->d_emb_tlen; E.text_cap = text_cap; E.next = c0; E.text_used = c1;
  cudaEvent_t* ev = ctx->stage_ev;
  if (kernel_ms) CK(cudaEventRecord(ev[0], st));
  CK(launch_emb_scan(E, ctx->sm_count, st));
  if (kernel_ms) CK(cudaEventRecord(ev[1], st));
  // the number of texts is only known on the device: read the row count back (4 bytes; the count kernel's grid is sized by it)
  unsigned int n_texts = 0;
  CK(cudaMemcpyAsync(&n_texts, c1, sizeof n_texts, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  // requests past the capacity were declined (AIGW_R_ARENA_FULL); every row below it was written in this call, the rows of a
  // request that straddles it as empty texts
  if (n_texts > text_cap) n_texts = text_cap;
  if (kernel_ms) CK(cudaEventRecord(ev[2], st));
  if (n_texts) {
    BpeParams P; P.text = d_bodies; P.offsets = ctx->d_emb_toff; P.lens = ctx->d_emb_tlen; P.n = n_texts; P.counts = ctx->d_emb_cnt; P.table = bpe->d_table; P.slots = bpe->slots; P.byte_to_id = bpe->d_b2i; P.next = c2;
    CK(launch_bpe_count(P, ctx->sm_count, st));
  }
  if (kernel_ms) CK(cudaEventRecord(ev[3], st));
  CK(launch_emb_sum(d_results, n, ctx->d_emb_cnt, st));
  if (kernel_ms) {
    CK(cudaEventRecord(ev[4], st)); CK(cudaEventSynchronize(ev[4]));
    CK(cudaEventElapsedTime(&kernel_ms[0], ev[0], ev[1])); CK(cudaEventElapsedTime(&kernel_ms[1], ev[2], ev[3])); CK(cudaEventElapsedTime(&kernel_ms[2], ev[3], ev[4])); CK(cudaEventElapsedTime(&kernel_ms[3], ev[0], ev[4]));
  }
  return 0;
}

int aigw_embeddings_count_host(aigw_ctx* ctx, const aigw_bpe* bpe, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n,
                               aigw_emb_count_result* results, uint64_t* h2d_bytes, uint64_t* d2h_bytes, float* kernel_ms) {
  if (!ctx || !bpe) return -2;
  if (n == 0) return 0;
  ENTER();
  uint32_t max_len = 0;
  for (uint32_t i = 0; i < n; i++) { if (lens[i] > max_len) max_len = lens[i]; if (offsets[i] & 15u) { ctx->err = "aigw_embeddings_count_host: request starts must be 16-byte aligned"; return -2; } }
  HostStage S(ctx);
  uint64_t nbytes = 0;
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n, &nbytes);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  aigw_emb_count_result* d_res = S.out<aigw_emb_count_result>(n);
  if (S.rc) return S.rc;
  if (int rc = aigw_embeddings_count_device(ctx, bpe, d_bodies, d_off, d_len, n, max_len, nbytes, d_res, S.st, kernel_ms)) return rc;
  S.back(results, d_res, n);
  S.d2h += 4;   // the device form's read-back of the text count
  return S.wait(h2d_bytes, d2h_bytes);
}

// ------------------------------------------------------------------ SSE
// ------------------------------------------------------------------ Cohere /v2/rerank requests of any size below 16 MiB
int aigw_rerank_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                       const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                       aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the cleaned ":path" and the override, exactly as the translate pass gets them
  RerankLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = (!cfg || cfg->schema != AIGW_SCHEMA_RERANK_COHERE) ? AIGW_R_SCHEMA : C.prefix_len == 0 ? AIGW_R_UNSUPPORTED_FIELD : 0;
  P.force_mutation = C.force_mutation ? 1u : 0u;
  P.override_len = C.override_len;
  P.override_ok = 1;
  for (uint32_t i = 0; i < C.override_len; i++) { const uint32_t c = (uint8_t)C.override_model[i]; if (c < 0x20 || c > 0x7f || c == '"' || c == '\\') P.override_ok = 0; }
  P.path_len = C.prefix_len;
  memcpy(P.override_model, C.override_model, sizeof P.override_model);
  memcpy(P.path, C.openai_path, sizeof P.path);
  P.tok_cap = rerank_tok_cap(max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u);
  const int grid = rerank_scan_grid(ctx->sm_count, P.tok_cap);
  CK(ctx->d_rr_tok.ensure((size_t)grid * P.tok_cap * 4));
  CK(ctx->d_rr_dep.ensure((size_t)grid * P.tok_cap));
  CK(ctx->d_rr_splice.ensure((size_t)n * sizeof(RerankSplice)));
  P.tok_ws = ctx->d_rr_tok; P.dep_ws = ctx->d_rr_dep; P.splice = ctx->d_rr_splice;
  unsigned int* c0;
  if (int rc = take_counters(ctx, 2, st, &c0)) return rc;
  P.next_scan = c0; P.next_emit = c0 + 1;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_rerank_large(P, ctx->sm_count, st)); return 0; });
}

int aigw_rerank_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                     const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (!ctx) return -2;
  if (n == 0) return 0;
  ENTER();
  ChatParams C;
  fill_params(C, cfg);
  // every record fits its slot: the path, the body, and the override with the ,"model":"" around it
  uint32_t max_len = 0;
  uint64_t cap = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i] & 15u) { ctx->err = "aigw_rerank_translate_large_host: request starts must be 16-byte aligned"; return -2; }
    if (lens[i] > max_len) max_len = lens[i];
    cap += ((uint64_t)C.prefix_len + lens[i] + C.override_len + 16u + 15u) & ~15ull;
  }
  HostStage S(ctx);
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  uint8_t* d_out = S.out<uint8_t>(cap);
  aigw_doc_result* d_res = S.out<aigw_doc_result>(n);
  uint64_t* d_used = S.out<uint64_t>(1);
  S.step([&] { CK(cudaMemsetAsync(d_used, 0, 8, S.st)); return 0; });
  S.step([&] { CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result))); CK(ctx->h_out.ensure(cap)); CK(ctx->h_used_arr.ensure(8)); return 0; });
  if (S.rc) return S.rc;
  float ms = 0;
  if (int rc = aigw_rerank_translate_large_device(ctx, cfg, d_bodies, d_off, d_len, n, max_len, d_out, cap, d_res, d_used, S.st, &ms)) return rc;
  S.back(ctx->h_res.p, d_res, n);
  S.back((uint64_t*)ctx->h_used_arr.p, d_used, 1);
  if (int rc = S.wait()) return rc;
  const uint64_t used = ctx->h_used_arr[0] < cap ? ctx->h_used_arr[0] : cap;
  if (used) { CK(cudaMemcpyAsync(ctx->h_out, d_out, used, cudaMemcpyDeviceToHost, S.st)); CK(cudaStreamSynchronize(S.st)); }
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = used; out->h2d_bytes = S.h2d + 8; out->d2h_bytes = S.d2h + used;
  out->gpu_launches = 2; out->kernel_ms = ms;
  return 0;
}

// ------------------------------------------------------------------ /v1/embeddings requests of any size below 16 MiB
int aigw_embeddings_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                           const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                           aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the ":path" prefix, override and api-version exactly as the translate pass gets them
  const int32_t schema = cfg ? cfg->schema : -1;
  const bool emb = schema == AIGW_SCHEMA_EMB_OPENAI || schema == AIGW_SCHEMA_EMB_AZURE_OPENAI || schema == AIGW_SCHEMA_EMB_GCP_VERTEX || schema == AIGW_SCHEMA_EMB_AWS_BEDROCK;
  EmbLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = emb ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.base = emb ? (uint32_t)(schema & 15) : 0u;
  P.force_mutation = C.force_mutation ? 1u : 0u;
  P.override_len = C.override_len;
  P.override_ok = 1;
  for (uint32_t i = 0; i < C.override_len; i++) { const uint32_t c = (uint8_t)C.override_model[i]; if (c < 0x20 || c > 0x7f || c == '"' || c == '\\') P.override_ok = 0; }
  emb_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.tok_cap = emb_tok_cap(ml); P.esc_cap = emb_esc_cap(ml); P.op_cap = emb_op_cap(ml);
  P.slice = emb_large_slice_bytes(ml);
  const int grid = emb_large_grid(ctx->sm_count, ml);
  CK(ctx->d_el_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_el_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_emb_large(P, grid, st)); return 0; });
}

using LargeDevice = int (*)(aigw_ctx*, const aigw_backend_cfg*, const uint8_t*, const uint64_t*, const uint32_t*, uint32_t, uint32_t, uint8_t*,
                            uint64_t, aigw_doc_result*, uint64_t*, void*, float*);

// The host form of a large-request device call whose records may exceed the first arena: Σ align16(path + k · len + 1024), the path
// bounded by the longest configuration path (or the model, at most the body).  A request whose record did not fit reports the
// length it needs, and those requests run once more into an arena of that size.
static int large_host_retry(LargeDevice dev, const char* name, uint32_t k, aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies,
                            const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (!ctx) return -2;
  if (n == 0) return 0;
  ENTER();
  ChatParams C;
  fill_params(C, cfg);
  const uint64_t path_max = (uint64_t)C.prefix_len + C.override_len + C.version_len + 64u;
  uint32_t max_len = 0;
  uint64_t cap = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i] & 15u) { ctx->err = std::string(name) + ": request starts must be 16-byte aligned"; return -2; }
    if (lens[i] > max_len) max_len = lens[i];
    cap += (path_max + (uint64_t)k * lens[i] + 1024u + 15u) & ~15ull;
  }
  HostStage S(ctx);
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  uint8_t* d_out = S.out<uint8_t>(cap);
  aigw_doc_result* d_res = S.out<aigw_doc_result>(n);
  uint64_t* d_used = S.out<uint64_t>(1);
  S.step([&] { CK(cudaMemsetAsync(d_used, 0, 8, S.st)); return 0; });
  S.step([&] { CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result))); CK(ctx->h_used_arr.ensure(8)); return 0; });
  if (S.rc) return S.rc;
  float ms = 0;
  if (int rc = dev(ctx, cfg, d_bodies, d_off, d_len, n, max_len, d_out, cap, d_res, d_used, S.st, &ms)) return rc;
  S.back(ctx->h_res.p, d_res, n);
  S.back((uint64_t*)ctx->h_used_arr.p, d_used, 1);
  if (int rc = S.wait()) return rc;
  uint64_t used = ctx->h_used_arr[0] < cap ? ctx->h_used_arr[0] : cap;
  uint64_t h2d = S.h2d + 8, d2h = S.d2h;
  uint32_t launches = 1;
  // requests whose record did not fit report the length they need (body_len): run them once more into an arena of that size
  std::vector<uint32_t> redo;
  uint64_t cap2 = 0;
  for (uint32_t i = 0; i < n; i++) {
    const aigw_doc_result& r = ctx->h_res[i];
    if (r.status == AIGW_DECLINED && r.reason == AIGW_R_OUT_SPACE && r.body_len) { redo.push_back(i); cap2 += ((uint64_t)r.body_len + 15u) & ~15ull; }
  }
  // the host arena holds the first run's records, then the second run's
  CK(ctx->h_out.ensure(used + cap2 + 16));
  if (used) CK(cudaMemcpyAsync(ctx->h_out, d_out, used, cudaMemcpyDeviceToHost, S.st));
  d2h += used;
  if (!redo.empty()) {
    // The retry stages into the first run's buffers (all but the bodies), and the first run's records are still being copied
    // out of one of them: wait for that copy before anything may reallocate or overwrite it.
    CK(cudaStreamSynchronize(S.st));
    const uint32_t m = (uint32_t)redo.size();
    std::vector<uint64_t> off2(m); std::vector<uint32_t> len2(m);
    for (uint32_t k = 0; k < m; k++) { off2[k] = offsets[redo[k]]; len2[k] = lens[redo[k]]; }
    HostStage S2(ctx);
    S2.next = 1;   // the bodies stay staged in the first buffer; the others are free again (the first run and its copy are complete)
    const uint64_t* d_off2 = S2.in(off2.data(), m);
    const uint32_t* d_len2 = S2.in(len2.data(), m);
    uint8_t* d_out2 = S2.out<uint8_t>(cap2);
    aigw_doc_result* d_res2 = S2.out<aigw_doc_result>(m);
    uint64_t* d_used2 = S2.out<uint64_t>(1);
    S2.step([&] { CK(cudaMemsetAsync(d_used2, 0, 8, S2.st)); return 0; });
    if (S2.rc) return S2.rc;
    uint32_t ml2 = 0; for (uint32_t k = 0; k < m; k++) if (len2[k] > ml2) ml2 = len2[k];
    float ms2 = 0;
    if (int rc = dev(ctx, cfg, d_bodies, d_off2, d_len2, m, ml2, d_out2, cap2, d_res2, d_used2, S2.st, &ms2)) return rc;
    std::vector<aigw_doc_result> res2(m);
    uint64_t used2 = 0;
    S2.back(res2.data(), d_res2, m);
    S2.back(&used2, d_used2, 1);
    if (int rc = S2.wait()) return rc;
    if (used2 > cap2) used2 = cap2;
    if (used2) CK(cudaMemcpyAsync(ctx->h_out.p + used, d_out2, used2, cudaMemcpyDeviceToHost, S2.st));
    CK(cudaStreamSynchronize(S2.st));
    for (uint32_t k = 0; k < m; k++) { aigw_doc_result r = res2[k]; if (r.status == AIGW_OK) r.out_off += used; ctx->h_res[redo[k]] = r; }
    h2d += S2.h2d + 8; d2h += S2.d2h + used2; used += used2; ms += ms2; launches++;
  } else CK(cudaStreamSynchronize(S.st));
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = used; out->h2d_bytes = h2d; out->d2h_bytes = d2h;
  out->gpu_launches = launches; out->kernel_ms = ms;
  return 0;
}

int aigw_embeddings_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                         const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  return large_host_retry(aigw_embeddings_translate_large_device, "aigw_embeddings_translate_large_host", 2, ctx, cfg, bodies, offsets, lens, n, out);
}

// ------------------------------------------------------------------ /v1/chat/completions passthroughs of any size below 16 MiB
int aigw_chat_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                     const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                     aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the ":path" prefix, override and api-version exactly as the translate pass gets them
  const int32_t schema = cfg ? cfg->schema : -1;
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = schema == AIGW_SCHEMA_OPENAI || schema == AIGW_SCHEMA_AZURE_OPENAI ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.azure = schema == AIGW_SCHEMA_AZURE_OPENAI ? 1u : 0u;
  P.cost_configured = C.cost_configured ? 1u : 0u;
  P.force_mutation = C.force_mutation ? 1u : 0u;
  P.override_len = C.override_len;
  P.override_ok = 1;
  for (uint32_t i = 0; i < C.override_len; i++) { const uint32_t c = (uint8_t)C.override_model[i]; if (c < 0x20 || c > 0x7f || c == '"' || c == '\\') P.override_ok = 0; }
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = chat_large_slice_bytes(ml);
  const int grid = chat_large_grid(ctx->sm_count, ml);
  CK(ctx->d_cl_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_cl_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_chat_large(P, grid, st)); return 0; });
}

int aigw_chat_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                   const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (!ctx) return -2;
  if (n == 0) return 0;
  ENTER();
  // output arena: Σ align16(2 · len + 512), which every record fits (the header states the bound)
  uint32_t max_len = 0;
  uint64_t cap = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i] & 15u) { ctx->err = "aigw_chat_translate_large_host: request starts must be 16-byte aligned"; return -2; }
    if (lens[i] > max_len) max_len = lens[i];
    cap += (2ull * lens[i] + 512u + 15u) & ~15ull;
  }
  HostStage S(ctx);
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  uint8_t* d_out = S.out<uint8_t>(cap);
  aigw_doc_result* d_res = S.out<aigw_doc_result>(n);
  uint64_t* d_used = S.out<uint64_t>(1);
  S.step([&] { CK(cudaMemsetAsync(d_used, 0, 8, S.st)); return 0; });
  S.step([&] { CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result))); CK(ctx->h_out.ensure(cap)); CK(ctx->h_used_arr.ensure(8)); return 0; });
  if (S.rc) return S.rc;
  float ms = 0;
  if (int rc = aigw_chat_translate_large_device(ctx, cfg, d_bodies, d_off, d_len, n, max_len, d_out, cap, d_res, d_used, S.st, &ms)) return rc;
  S.back(ctx->h_res.p, d_res, n);
  S.back((uint64_t*)ctx->h_used_arr.p, d_used, 1);
  if (int rc = S.wait()) return rc;
  const uint64_t used = ctx->h_used_arr[0] < cap ? ctx->h_used_arr[0] : cap;
  if (used) { CK(cudaMemcpyAsync(ctx->h_out, d_out, used, cudaMemcpyDeviceToHost, S.st)); CK(cudaStreamSynchronize(S.st)); }
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = used; out->h2d_bytes = S.h2d + 8; out->d2h_bytes = S.d2h + used;
  out->gpu_launches = 1; out->kernel_ms = ms;
  return 0;
}

// ------------------------------------------------------------------ /v1/chat/completions to AWS Bedrock Converse of any size below 16 MiB
int aigw_chat_bedrock_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                             const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                             aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the override exactly as the translate pass gets it
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = cfg && cfg->schema == AIGW_SCHEMA_AWS_BEDROCK ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.azure = 0; P.cost_configured = 0; P.force_mutation = 0; P.override_ok = 1;   // the Converse body is always rebuilt
  P.override_len = C.override_len;
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.max_len = ml;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = chat_record_large_slice_bytes(ml);
  const int grid = chat_record_large_grid(ctx->sm_count, ml);
  CK(ctx->d_bl_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_bl_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_chat_bedrock_large(P, grid, st)); return 0; });
}

int aigw_chat_bedrock_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                           const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  return large_host_retry(aigw_chat_bedrock_translate_large_device, "aigw_chat_bedrock_translate_large_host", 3, ctx, cfg, bodies, offsets, lens, n, out);
}

// ------------------------------------------------------------------ /v1/chat/completions to Anthropic on GCP Vertex AI / AWS Bedrock of any size below 16 MiB
int aigw_chat_anthropic_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                               const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                               aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the override and api-version exactly as the translate pass gets them
  const int32_t schema = cfg ? cfg->schema : -1;
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = schema == AIGW_SCHEMA_GCP_ANTHROPIC || schema == AIGW_SCHEMA_AWS_ANTHROPIC ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.gcp = schema == AIGW_SCHEMA_GCP_ANTHROPIC ? 1u : 0u;
  P.azure = 0; P.cost_configured = 0; P.force_mutation = 0; P.override_ok = 1;   // the Messages body is always rebuilt
  P.override_len = C.override_len;
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.max_len = ml;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = chat_record_large_slice_bytes(ml);
  const int grid = chat_record_large_grid(ctx->sm_count, ml);
  CK(ctx->d_al_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_al_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_chat_anthropic_large(P, grid, st)); return 0; });
}

int aigw_chat_anthropic_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                             const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  // the densest record is a run of the shortest tool messages ({"content":"x","role":"tool"}, 30 bytes with its comma, become
  // 96-byte tool_result blocks): 3.2 times the body
  return large_host_retry(aigw_chat_anthropic_translate_large_device, "aigw_chat_anthropic_translate_large_host", 4, ctx, cfg, bodies, offsets, lens, n, out);
}

// ------------------------------------------------------------------ /v1/chat/completions to Gemini on GCP Vertex AI of any size below 16 MiB
int aigw_chat_gemini_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                            const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                            aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the override exactly as the translate pass gets it
  const int32_t schema = cfg ? cfg->schema : -1;
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = schema == AIGW_SCHEMA_GCP_VERTEX ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.gcp = 0; P.azure = 0; P.cost_configured = 0; P.force_mutation = 0; P.override_ok = 1;   // the GenerateContent body is always rebuilt
  P.override_len = C.override_len;
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.max_len = ml;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = chat_record_large_slice_bytes(ml);
  const int grid = chat_record_large_grid(ctx->sm_count, ml);
  CK(ctx->d_al_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_al_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_chat_gemini_large(P, grid, st)); return 0; });
}

int aigw_chat_gemini_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                          const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  // the densest record is a user text of backslash-b escapes (two bytes each, re-spelled as six-byte u-escapes): 3.0 times the body
  return large_host_retry(aigw_chat_gemini_translate_large_device, "aigw_chat_gemini_translate_large_host", 3, ctx, cfg, bodies, offsets, lens, n, out);
}

// ------------------------------------------------------------------ /v1/messages to OpenAI and AWS Bedrock Converse of any size below 16 MiB
int aigw_messages_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                         const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                         aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the ":path" prefix and the override exactly as the translate pass gets them
  const int32_t schema = cfg ? cfg->schema : -1;
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = schema == AIGW_SCHEMA_MSG_OPENAI || schema == AIGW_SCHEMA_MSG_AWS_BEDROCK ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.bedrock = schema == AIGW_SCHEMA_MSG_AWS_BEDROCK ? 1u : 0u;
  P.gcp = 0; P.azure = 0; P.cost_configured = 0; P.force_mutation = 0; P.override_ok = 1;   // the body is always rebuilt
  P.override_len = C.override_len;
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.max_len = ml;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = chat_record_large_slice_bytes(ml);
  const int grid = chat_record_large_grid(ctx->sm_count, ml);
  CK(ctx->d_al_ws.ensure((size_t)grid * P.slice));
  P.ws = ctx->d_al_ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_messages_large(P, grid, st)); return 0; });
}

int aigw_messages_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                       const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  // the densest record is a text of backslash-b escapes (two bytes each, re-spelled as six-byte u-escapes): 3.0 times the body
  return large_host_retry(aigw_messages_translate_large_device, "aigw_messages_translate_large_host", 3, ctx, cfg, bodies, offsets, lens, n, out);
}

// ------------------------------------------------------------------ /v1/responses and /v1/completions requests of any size below 16 MiB
// The OpenAI passthroughs whose ParseBody returns no mutated body: one kernel per schema on ChatLargeParams, each with its own
// slice size, grid and context workspace.
struct OpenAILarge {
  int32_t schema;
  const char* host_name;   // for the alignment error
  uint64_t (*slice_bytes)(uint32_t);
  int (*grid)(int, uint32_t);
  cudaError_t (*launch)(const ChatLargeParams&, int, cudaStream_t);
  Scratch<uint8_t> aigw_ctx::*ws;
};
static const OpenAILarge kResponsesLarge = {AIGW_SCHEMA_RESPONSES_OPENAI, "aigw_responses_translate_large_host", responses_large_slice_bytes,
                                            responses_large_grid, launch_responses_large, &aigw_ctx::d_rl_ws};
static const OpenAILarge kCompletionsLarge = {AIGW_SCHEMA_COMPLETIONS_OPENAI, "aigw_completions_translate_large_host", completions_large_slice_bytes,
                                              completions_large_grid, launch_completions_large, &aigw_ctx::d_cpl_ws};

static int openai_large_device(const OpenAILarge& K, aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                               const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                               aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (!ctx) return -2;
  if (n == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  ChatParams C;
  fill_params(C, cfg);   // the ":path" (path.Join("/", prefix, "responses" / "completions")) and the override exactly as the translate pass gets them
  ChatLargeParams P;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.results = d_results;
  P.out = d_out; P.out_capacity = out_capacity; P.out_used = (unsigned long long*)d_out_used;
  P.call_reason = cfg && cfg->schema == K.schema ? 0u : (uint32_t)AIGW_R_SCHEMA;
  P.azure = 0; P.cost_configured = 0;   // one backend; ParseBody forces no include_usage here
  P.force_mutation = C.force_mutation ? 1u : 0u;
  P.override_len = C.override_len;
  P.override_ok = 1;
  for (uint32_t i = 0; i < C.override_len; i++) { const uint32_t c = (uint8_t)C.override_model[i]; if (c < 0x20 || c > 0x7f || c == '"' || c == '\\') P.override_ok = 0; }
  chat_large_lits(P, C.openai_path, C.prefix_len, C.override_model, C.override_len, C.api_version, C.version_len);
  const uint32_t ml = max_len && max_len < (1u << 24) ? max_len : (1u << 24) - 1u;
  P.tok_cap = chat_large_tok_cap(ml);
  P.slice = K.slice_bytes(ml);
  const int grid = K.grid(ctx->sm_count, ml);
  Scratch<uint8_t>& ws = ctx->*K.ws;
  CK(ws.ensure((size_t)grid * P.slice));
  P.ws = ws;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(K.launch(P, grid, st)); return 0; });
}

static int openai_large_host(const OpenAILarge& K, aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                             const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (!ctx) return -2;
  if (n == 0) return 0;
  ENTER();
  ChatParams C;
  fill_params(C, cfg);
  // every record fits its slot: the path, the body, and the override with the ,"model":"" around it
  uint32_t max_len = 0;
  uint64_t cap = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i] & 15u) { ctx->err = std::string(K.host_name) + ": request starts must be 16-byte aligned"; return -2; }
    if (lens[i] > max_len) max_len = lens[i];
    cap += ((uint64_t)C.prefix_len + lens[i] + C.override_len + 16u + 15u) & ~15ull;
  }
  HostStage S(ctx);
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n);
  const uint64_t* d_off = S.in(offsets, n);
  const uint32_t* d_len = S.in(lens, n);
  uint8_t* d_out = S.out<uint8_t>(cap);
  aigw_doc_result* d_res = S.out<aigw_doc_result>(n);
  uint64_t* d_used = S.out<uint64_t>(1);
  S.step([&] { CK(cudaMemsetAsync(d_used, 0, 8, S.st)); return 0; });
  S.step([&] { CK(ctx->h_res.ensure((size_t)n * sizeof(aigw_doc_result))); CK(ctx->h_out.ensure(cap)); CK(ctx->h_used_arr.ensure(8)); return 0; });
  if (S.rc) return S.rc;
  float ms = 0;
  if (int rc = openai_large_device(K, ctx, cfg, d_bodies, d_off, d_len, n, max_len, d_out, cap, d_res, d_used, S.st, &ms)) return rc;
  S.back(ctx->h_res.p, d_res, n);
  S.back((uint64_t*)ctx->h_used_arr.p, d_used, 1);
  if (int rc = S.wait()) return rc;
  const uint64_t used = ctx->h_used_arr[0] < cap ? ctx->h_used_arr[0] : cap;
  if (used) { CK(cudaMemcpyAsync(ctx->h_out, d_out, used, cudaMemcpyDeviceToHost, S.st)); CK(cudaStreamSynchronize(S.st)); }
  out->results = ctx->h_res; out->out = ctx->h_out; out->out_used = used; out->h2d_bytes = S.h2d + 8; out->d2h_bytes = S.d2h + used;
  out->gpu_launches = 1; out->kernel_ms = ms;
  return 0;
}

int aigw_responses_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                          const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                          aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  return openai_large_device(kResponsesLarge, ctx, cfg, d_bodies, d_offsets, d_lens, n, max_len, d_out, out_capacity, d_results, d_out_used, stream, kernel_ms);
}

int aigw_responses_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                        const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  return openai_large_host(kResponsesLarge, ctx, cfg, bodies, offsets, lens, n, out);
}

int aigw_completions_translate_large_device(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* d_bodies, const uint64_t* d_offsets,
                                            const uint32_t* d_lens, uint32_t n, uint32_t max_len, uint8_t* d_out, uint64_t out_capacity,
                                            aigw_doc_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  return openai_large_device(kCompletionsLarge, ctx, cfg, d_bodies, d_offsets, d_lens, n, max_len, d_out, out_capacity, d_results, d_out_used, stream, kernel_ms);
}

int aigw_completions_translate_large_host(aigw_ctx* ctx, const aigw_backend_cfg* cfg, const uint8_t* bodies, const uint64_t* offsets,
                                          const uint32_t* lens, uint32_t n, aigw_batch_out* out) {
  return openai_large_host(kCompletionsLarge, ctx, cfg, bodies, offsets, lens, n, out);
}

int aigw_sse_usage_device(aigw_ctx* ctx, const uint8_t* d_bytes, const uint64_t* d_chunk_off, const uint32_t* d_chunk_first,
                          uint32_t n_streams, aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  if (n_streams == 0) { if (kernel_ms) *kernel_ms = 0; return 0; }
  ENTER_ON(stream);
  SseParams P; P.bytes = d_bytes; P.chunk_off = d_chunk_off; P.chunk_first = d_chunk_first; P.n_streams = n_streams; P.results = d_results;
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_sse_usage(P, ctx->sm_count, st)); return 0; });
}

int aigw_sse_usage_host(aigw_ctx* ctx, const uint8_t* bytes, const uint64_t* chunk_off, const uint32_t* chunk_first,
                        uint32_t n_streams, uint32_t n_chunks, aigw_sse_result* results, uint64_t* h2d_bytes, uint64_t* d2h_bytes, float* kernel_ms) {
  if (n_streams == 0) return 0;
  ENTER();
  HostStage S(ctx);
  const uint8_t* d_bytes = S.in(bytes, chunk_off[n_chunks]);
  const uint64_t* d_chunk_off = S.in(chunk_off, (size_t)n_chunks + 1);
  const uint32_t* d_chunk_first = S.in(chunk_first, (size_t)n_streams + 1);
  aigw_sse_result* d_res = S.out<aigw_sse_result>(n_streams);
  if (S.rc) return S.rc;
  if (int rc = aigw_sse_usage_device(ctx, d_bytes, d_chunk_off, d_chunk_first, n_streams, d_res, S.st, kernel_ms)) return rc;
  S.back(results, d_res, n_streams);
  return S.wait(h2d_bytes, d2h_bytes);
}

// ------------------------------------------------------------------ stateful per-chunk response streams
static int stream_pool_grow(aigw_ctx* ctx, uint32_t want) {
  auto& sp = ctx->sp;
  if (want <= sp.cap) return 0;
  uint32_t ncap = sp.cap ? sp.cap : 1024u;
  while (ncap < want) ncap *= 2;
  if (ncap > (1u << 22)) { ctx->err = "too many open streams"; return -3; }
  Scratch<StreamSlot> nd;   // copy, then swap: the old slots are freed with nd, and so is nd when the copy fails
  CK(nd.ensure((size_t)ncap * sizeof(StreamSlot)));
  if (sp.cap) { CK(cudaMemcpyAsync(nd, sp.d_slots, (size_t)sp.cap * sizeof(StreamSlot), cudaMemcpyDeviceToDevice, ctx->s_compute)); CK(cudaStreamSynchronize(ctx->s_compute)); }
  sp.d_slots.swap(nd);
  sp.carry.resize(ncap, 0); sp.gen.resize(ncap, 0); sp.stamp.resize(ncap, 0); sp.open.resize(ncap, 0); sp.kind.resize(ncap, 0); sp.model_len.resize(ncap, 0);
  for (uint32_t i = ncap; i-- > sp.cap;) sp.free_list.push_back(i);
  sp.cap = ncap;
  return 0;
}
static bool stream_handle_ok(aigw_ctx* ctx, uint64_t h, uint32_t& slot) {
  auto& sp = ctx->sp;
  const uint32_t lo = (uint32_t)h; if (lo == 0 || lo > sp.cap) return false;
  slot = lo - 1;
  return sp.open[slot] && sp.gen[slot] == (uint32_t)(h >> 32);
}

int aigw_stream_open_batch(aigw_ctx* ctx, const aigw_stream_cfg* cfg, uint32_t n, uint64_t* handles) {
  if (!cfg || (n && !handles)) return -2;
  if (n == 0) return 0;
  ENTER();
  auto& sp = ctx->sp;
  std::lock_guard<std::mutex> lk(sp.mu);
  const char* model = cfg->request_model ? cfg->request_model : ""; const char* id = cfg->response_id ? cfg->response_id : "";
  if (cfg->kind < AIGW_STREAM_OPENAI || cfg->kind > AIGW_STREAM_OPENAI_RESPONSES || strlen(model) > 160 || strlen(id) > 160 || !plain_json_text(model) || !plain_json_text(id)) {
    ctx->err = "stream cfg: unknown kind, or request_model / response_id need JSON escaping or exceed 160 bytes"; return -2;
  }
  if (sp.free_list.size() < n) { const int rc = stream_pool_grow(ctx, sp.cap + (uint32_t)(n - sp.free_list.size())); if (rc) return rc; }
  std::vector<uint8_t> tmpl(kStreamHdrBytes, 0);
  StreamSlot* t = (StreamSlot*)tmpl.data();   // header part only
  t->kind = (uint32_t)cfg->kind; t->beg = t->end = 0; t->flags = 0; t->tool_index = cfg->kind == AIGW_STREAM_GCP_ANTHROPIC ? -1 : 0; t->active_index = -1;
  t->created = cfg->created; t->model_len = (uint32_t)strlen(model); memcpy(t->model, model, t->model_len);
  if (cfg->kind == AIGW_STREAM_AWS_BEDROCK) { t->id_len = (uint32_t)strlen(id); memcpy(t->id, id, t->id_len); t->flags |= SF_HAVE_CREATED; }
  CK(sp.d_tmpl.ensure(kStreamHdrBytes));
  CK(sp.d_ids.ensure((size_t)n * 4));
  CK(sp.h_ids.ensure((size_t)n * 4));
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t slot = sp.free_list.back(); sp.free_list.pop_back();
    sp.open[slot] = 1; sp.gen[slot]++; sp.carry[slot] = 0; sp.kind[slot] = t->kind; sp.model_len[slot] = t->model_len;
    sp.h_ids[i] = slot; handles[i] = ((uint64_t)sp.gen[slot] << 32) | (uint64_t)(slot + 1);
  }
  cudaStream_t st = ctx->s_compute;
  CK(cudaMemcpyAsync(sp.d_tmpl, tmpl.data(), kStreamHdrBytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(sp.d_ids, sp.h_ids, (size_t)n * 4, cudaMemcpyHostToDevice, st));
  CK(launch_stream_init(sp.d_slots, sp.d_ids, n, sp.d_tmpl, st));
  CK(cudaStreamSynchronize(st));
  return 0;
}
int aigw_stream_open(aigw_ctx* ctx, const aigw_stream_cfg* cfg, uint64_t* handle) { return aigw_stream_open_batch(ctx, cfg, 1, handle); }

int aigw_stream_close_batch(aigw_ctx* ctx, const uint64_t* handles, uint32_t n) {
  auto& sp = ctx->sp;
  std::lock_guard<std::mutex> lk(sp.mu);
  int rc = 0;
  for (uint32_t i = 0; i < n; i++) { uint32_t slot; if (!stream_handle_ok(ctx, handles[i], slot)) { rc = -2; continue; } sp.open[slot] = 0; sp.free_list.push_back(slot); }
  return rc;
}
int aigw_stream_close(aigw_ctx* ctx, uint64_t handle) { return aigw_stream_close_batch(ctx, &handle, 1); }

// One window of ResponseBody calls.  get(i) = {handle, bytes, len, eos} of call i.  zc_base != nullptr: every call's bytes lie in one
// mapped pinned buffer starting at zc_base (device view zc_dev): the kernels read them in place, nothing is staged or copied.
extern "C++" {
struct StreamCallIn { uint64_t handle; const uint8_t* bytes; uint32_t len; uint32_t eos; };
template <class GET>
static int stream_chunks_core(aigw_ctx* ctx, uint32_t n, GET&& get, aigw_chunk_result* results, const uint8_t** arena, const uint8_t* zc_base, const uint8_t* zc_dev) {
  auto& sp = ctx->sp;
  if (arena) *arena = nullptr;
  if (n == 0) return 0;
  static const bool prof = getenv("AIGW_STREAM_PROF") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
  const auto t0 = now();
  CK(sp.h_steps.ensure((size_t)n * sizeof(StreamStep)));
  sp.call_no++;
  uint64_t in_bytes = 0, out_bytes = 0;
  for (uint32_t i = 0; i < n; i++) {
    const StreamCallIn c = get(i);
    uint32_t slot;
    if (!stream_handle_ok(ctx, c.handle, slot) || (c.len && !c.bytes)) { ctx->err = "aigw_stream_chunks: bad handle"; return -2; }
    if (sp.stamp[slot] == sp.call_no) { ctx->err = "aigw_stream_chunks: a stream appears twice in one call"; return -2; }
    sp.stamp[slot] = sp.call_no;
    StreamStep& s = sp.h_steps[i];
    s.slot = slot; s.len = c.len; s.eos = c.eos ? 1u : 0u;
    if (zc_base) s.in_off = (uint64_t)(c.bytes - zc_base);
    else { s.in_off = in_bytes; in_bytes += ((uint64_t)c.len + 15u) & ~15ull; }
    s.out_cap = stream_out_cap(sp.kind[slot], (uint64_t)sp.carry[slot] + c.len, sp.model_len[slot]);
    s.out_off = out_bytes; out_bytes += ((uint64_t)s.out_cap + 15u) & ~15ull;
  }
  if (!zc_base) { CK(sp.h_in.ensure(in_bytes + 16)); CK(sp.d_in.ensure(in_bytes + 16)); }
  CK(sp.d_steps.ensure((size_t)n * sizeof(StreamStep)));
  CK(sp.d_res.ensure((size_t)n * sizeof(aigw_chunk_result)));
  CK(sp.h_res.ensure((size_t)n * sizeof(aigw_chunk_result)));
  CK(sp.d_out.ensure(out_bytes + 16));
  CK(sp.d_packed.ensure(out_bytes + 16));
  CK(sp.d_used.ensure(8)); CK(sp.h_used.ensure(8));
  const auto t1 = now();
  if (!zc_base) host_parallel_for(n, [&](uint32_t b, uint32_t e) { for (uint32_t i = b; i < e; i++) { const StreamCallIn c = get(i); if (c.len) memcpy(sp.h_in + sp.h_steps[i].in_off, c.bytes, c.len); } });   // no caller pointer is retained
  const auto t2 = now();
  cudaStream_t st = ctx->s_compute;
  if (!zc_base) CK(cudaMemcpyAsync(sp.d_in, sp.h_in, in_bytes, cudaMemcpyHostToDevice, st));
  CK(cudaMemcpyAsync(sp.d_steps, sp.h_steps, (size_t)n * sizeof(StreamStep), cudaMemcpyHostToDevice, st));
  CK(cudaMemsetAsync(sp.d_used, 0, 8, st));
  StreamParams P; P.slots = sp.d_slots; P.in = zc_base ? zc_dev : sp.d_in; P.out = sp.d_out; P.packed = sp.d_packed; P.packed_used = sp.d_used; P.packed_cap = sp.d_packed.cap; P.steps = sp.d_steps; P.results = sp.d_res; P.n = n;
  CK(launch_stream_steps(P, st));
  // results: straight into the caller's array when it is pinned (one DMA), else through the pinned staging array
  cudaPointerAttributes ra; const bool res_pinned = cudaPointerGetAttributes(&ra, results) == cudaSuccess && ra.type == cudaMemoryTypeHost;
  if (!res_pinned) cudaGetLastError();
  aigw_chunk_result* hres = res_pinned ? results : sp.h_res;
  CK(cudaMemcpyAsync(hres, sp.d_res, (size_t)n * sizeof(aigw_chunk_result), cudaMemcpyDeviceToHost, st));
  CK(cudaMemcpyAsync(sp.h_used, sp.d_used, 8, cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  const auto t3 = now();
  const uint64_t used = *sp.h_used < sp.d_packed.cap ? *sp.h_used : sp.d_packed.cap;
  if (used) {
    CK(sp.h_packed.ensure(used + 16));
    CK(cudaMemcpyAsync(sp.h_packed, sp.d_packed, used, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
  }
  const auto t4 = now();
  if (res_pinned) { for (uint32_t i = 0; i < n; i++) sp.carry[sp.h_steps[i].slot] = results[i].carry_len; }
  else host_parallel_for(n, [&](uint32_t b, uint32_t e) { for (uint32_t i = b; i < e; i++) { results[i] = sp.h_res[i]; sp.carry[sp.h_steps[i].slot] = sp.h_res[i].carry_len; } });   // a stream appears once per call: the carry writes are disjoint
  if (arena) *arena = sp.h_packed;
  if (prof && (sp.call_no & 63) == 1) fprintf(stderr, "stream_chunks n=%u%s: table %.0f us, byte staging %.0f us, H2D + kernels + D2H results %.0f us, D2H packed %.0f us, result copy %.0f us\n", n, zc_base ? " (zero-copy input)" : "", us(t0, t1), us(t1, t2), us(t2, t3), us(t3, t4), us(t4, now()));
  return 0;
}
}  // extern "C++"
int aigw_stream_chunks(aigw_ctx* ctx, const aigw_chunk_in* in, uint32_t n, aigw_chunk_result* results, const uint8_t** arena) {
  ENTER();
  std::lock_guard<std::mutex> lk(ctx->sp.mu);
  return stream_chunks_core(ctx, n, [&](uint32_t i) { return StreamCallIn{in[i].handle, in[i].bytes, in[i].len, in[i].eos}; }, results, arena, nullptr, nullptr);
}
/* structure-of-arrays form: chunk i of the call = base[off[i] .. off[i]+len[i]) for stream handles[i] (batch drivers, bench config 4).
 * When `base` is mapped pinned memory (aigw_host_alloc) the kernels read the chunks in place: no staging copy, no H2D of the bytes. */
int aigw_stream_chunks_soa(aigw_ctx* ctx, const uint64_t* handles, const uint8_t* base, const uint64_t* off, const uint32_t* len, const uint8_t* eos, uint32_t n,
                           aigw_chunk_result* results, const uint8_t** arena) {
  ENTER();
  std::lock_guard<std::mutex> lk(ctx->sp.mu);
  const uint8_t* zc_dev = nullptr;
  {
    static const bool no_zc = getenv("AIGW_STREAM_NO_ZEROCOPY") != nullptr;
    cudaPointerAttributes at;
    if (!no_zc && base && cudaPointerGetAttributes(&at, base) == cudaSuccess && at.type == cudaMemoryTypeHost && at.devicePointer) zc_dev = (const uint8_t*)at.devicePointer;
    else cudaGetLastError();
  }
  return stream_chunks_core(ctx, n, [&](uint32_t i) { return StreamCallIn{handles[i], base + off[i], len[i], eos ? (uint32_t)eos[i] : 0u}; }, results, arena, zc_dev ? base : nullptr, zc_dev);
}
int aigw_stream_chunk(aigw_ctx* ctx, uint64_t handle, const uint8_t* bytes, uint32_t len, int eos, uint8_t* out, uint32_t out_cap, aigw_chunk_result* res) {
  ENTER();
  std::lock_guard<std::mutex> lk(ctx->sp.mu);
  aigw_chunk_in in; in.handle = handle; in.bytes = bytes; in.len = len; in.eos = eos ? 1u : 0u;
  const uint8_t* arena = nullptr;
  const int rc = stream_chunks_core(ctx, 1, [&](uint32_t) { return StreamCallIn{in.handle, in.bytes, in.len, in.eos}; }, res, &arena, nullptr, nullptr);
  if (rc) return rc;
  const uint32_t tot = res->out_len + res->model_len;
  if (tot > out_cap) return -4;
  if (tot) memcpy(out, arena + res->out_off, tot);
  res->out_off = 0;
  return 0;
}

// ------------------------------------------------------------------ S2: Bedrock eventstream → OpenAI SSE
static int fill_stream_params(aigw_ctx* ctx, BedrockStreamParams& P, const aigw_bedrock_stream_cfg* cfg) {
  memset(P.id, 0, sizeof P.id); memset(P.model, 0, sizeof P.model); P.id_len = P.model_len = 0; P.created = cfg ? cfg->created : 0;
  const char* id = cfg && cfg->response_id ? cfg->response_id : ""; const char* model = cfg && cfg->request_model ? cfg->request_model : "";
  if (strlen(id) > sizeof P.id || strlen(model) > sizeof P.model || !plain_json_text(id) || !plain_json_text(model)) { ctx->err = "response_id/request_model need JSON escaping or exceed 128 bytes"; return -2; }
  P.id_len = (uint32_t)strlen(id); memcpy(P.id, id, P.id_len); P.model_len = (uint32_t)strlen(model); memcpy(P.model, model, P.model_len);
  return 0;
}
// one batch of streams on st, P's buffers set and d_bs_work large enough: the device form, and each chunk of the host form
static int bedrock_stream_device_impl(aigw_ctx* ctx, BedrockStreamParams& P, cudaStream_t st, float* kernel_ms) {
  bedrock_work_layout(P, ctx->d_bs_work, P.n_streams);
  if (int rc = take_counters(ctx, 2, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_bedrock_stream(P, ctx->sm_count, st)); return 0; });
}
int aigw_bedrock_stream_device(aigw_ctx* ctx, const aigw_bedrock_stream_cfg* cfg, const uint8_t* d_bytes, const uint64_t* d_stream_off, uint32_t n_streams,
                               uint64_t total_bytes, uint8_t* d_out, uint64_t out_capacity, aigw_stream_result* d_results, uint64_t* d_out_used,
                               void* stream, float* kernel_ms) {
  if (kernel_ms) *kernel_ms = 0;
  if (n_streams == 0) return 0;
  ENTER_ON(stream);
  BedrockStreamParams P;
  if (int rc = fill_stream_params(ctx, P, cfg)) return rc;
  CK(ctx->d_bs_work.ensure(bedrock_work_bytes(total_bytes, n_streams)));
  P.bytes = d_bytes; P.stream_off = d_stream_off; P.off_base = 0; P.out_bias = 0; P.n_streams = n_streams; P.out = d_out; P.out_capacity = out_capacity; P.results = d_results;
  P.out_used = (unsigned long long*)d_out_used;
  CK(cudaMemsetAsync(d_out_used, 0, sizeof(uint64_t), st));
  return bedrock_stream_device_impl(ctx, P, st, kernel_ms);
}

int aigw_bedrock_stream_host(aigw_ctx* ctx, const aigw_bedrock_stream_cfg* cfg, const uint8_t* bytes, const uint64_t* stream_off, uint32_t n_streams,
                             uint64_t out_capacity_hint, aigw_stream_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (n_streams == 0) return 0;
  ENTER();
  BedrockStreamParams P0;
  if (int rc = fill_stream_params(ctx, P0, cfg)) return rc;
  const uint64_t total_in = stream_off[n_streams] - stream_off[0];
  const double ratio = out_capacity_hint ? (double)out_capacity_hint / (double)(total_in + 1) : 2.0;
  return chunk_pipeline(
      ctx, bytes, stream_off, nullptr, n_streams, 64ull << 20,
      [&](uint64_t ib, uint32_t nd) { return ((uint64_t)((double)ib * ratio) + (uint64_t)nd * 64 + 4096 + 255) & ~255ull; }, 2,
      [&](const PipeChunk<aigw_stream_result>& k) {
        CK(ctx->d_bs_work.ensure(bedrock_work_bytes(k.max_in, k.max_n)));   // the chunks share it: sized once, by the first
        BedrockStreamParams P = P0;
        P.bytes = k.bytes; P.stream_off = k.off; P.off_base = stream_off[k.first]; P.n_streams = k.n;
        P.out = k.out; P.out_capacity = k.out_cap; P.out_bias = k.out_bias; P.results = k.results; P.out_used = k.out_used;
        return bedrock_stream_device_impl(ctx, P, ctx->s_compute, nullptr);
      },
      out);
}

// ------------------------------------------------------------------ B1: body mutation
static bool mut_path_ok(const char* p) {
  bool digits = true;
  for (const char* q = p; *q; q++) {
    const unsigned char c = (unsigned char)*q;
    if (c == '.' || c == '*' || c == '?' || c == '#' || c == '|' || c == ':' || c == '\\' || c == '@' || c < 0x21 || c > 0x7e || c == '"') return false;
    if (c < '0' || c > '9') digits = false;
  }
  return !digits && strcmp(p, "-1") != 0;
}
// isJSONValue (internal/bodymutator/body_mutator.go:33-75)
static bool mut_is_json_value(const std::string& value) {
  size_t b = 0, e = value.size();
  auto sp = [](unsigned char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r' || c == 0x85 || c == 0xA0; };
  while (b < e && sp((unsigned char)value[b])) b++;
  while (e > b && sp((unsigned char)value[e - 1])) e--;
  const std::string v = value.substr(b, e - b);
  if (!v.empty() && v.front() == '"' && v.back() == '"') return true;
  if (v == "0" || v == "true" || v == "false" || v == "null") return true;
  if (!v.empty()) {
    const char f = v[0];
    if ((f >= '0' && f <= '9') || f == '-' || f == '+') {
      bool num = true;
      for (char c : v) if ((c < '0' || c > '9') && c != '.' && c != '-' && c != '+' && c != 'e' && c != 'E') { num = false; break; }
      if (num) return true;
    }
  }
  if (!v.empty() && v.front() == '{' && v.back() == '}') return true;
  if (!v.empty() && v.front() == '[' && v.back() == ']') return true;
  return false;
}
// fold the configured remove / set lists into per-key actions (see mutate_kernel.cuh)
static int fill_mutate_params(aigw_ctx* ctx, MutateParams& P, const aigw_body_mutation* m) {
  memset(P.keys, 0, sizeof P.keys); memset(P.text, 0, sizeof P.text); P.n_keys = 0;
  P.text[kMutTextCap - 4] = ',';
  struct K { std::string name, raw; bool remove = false, set = false; };
  std::vector<K> keys;
  auto find = [&](const char* name) -> K* { for (auto& k : keys) if (k.name == name) return &k; return nullptr; };
  for (uint32_t i = 0; m && i < m->n_set; i++) {
    const char* path = m->set[i].path; const char* val = m->set[i].value ? m->set[i].value : "";
    if (!path || !*path) continue;
    if (!mut_path_ok(path)) { ctx->err = std::string("body mutation path is not a plain top-level key: ") + path; return -2; }
    std::string raw;
    if (mut_is_json_value(val)) raw = val;
    else {   // sjson.SetBytes of a Go string: plain quoting when nothing needs escaping
      for (const char* q = val; *q; q++) { const unsigned char c = (unsigned char)*q; if (c < ' ' || c > 0x7f || c == '"' || c == '\\') { ctx->err = std::string("body mutation value needs JSON escaping: ") + path; return -2; } }
      raw = std::string("\"") + val + "\"";
    }
    K* k = find(path);
    if (!k) { keys.push_back(K{}); k = &keys.back(); k->name = path; }
    k->set = true; k->raw = raw;
  }
  for (uint32_t i = 0; m && i < m->n_remove; i++) {
    const char* path = m->remove[i];
    if (!path || !*path) continue;
    if (!mut_path_ok(path)) { ctx->err = std::string("body mutation path is not a plain top-level key: ") + path; return -2; }
    K* k = find(path);
    if (!k) { keys.push_back(K{}); k = &keys.back(); k->name = path; }
    k->remove = true;
  }
  if (keys.size() > (size_t)kMutMaxKeys) { ctx->err = "more than 16 distinct body mutation keys"; return -2; }
  size_t o = 0;
  for (size_t i = 0; i < keys.size(); i++) {
    const K& k = keys[i]; MutateKey& mk = P.keys[i];
    const std::string memb = "\"" + k.name + "\":" + k.raw;
    if (o + k.name.size() + memb.size() + 8 > (size_t)kMutTextCap - 8) { ctx->err = "body mutation text exceeds 3 KiB"; return -2; }
    mk.name_off = (uint16_t)o; mk.name_len = (uint16_t)k.name.size(); memcpy(P.text + o, k.name.data(), k.name.size()); o += (k.name.size() + 3) & ~(size_t)3;
    mk.memb_off = (uint16_t)o; mk.memb_len = (uint16_t)memb.size(); memcpy(P.text + o, memb.data(), memb.size());
    mk.val_off = (uint16_t)(o + k.name.size() + 3); mk.val_len = (uint16_t)k.raw.size();
    o += (memb.size() + 3) & ~(size_t)3;
    mk.remove = k.remove; mk.set = k.set;
  }
  P.n_keys = (uint32_t)keys.size();
  return 0;
}
// one batch of bodies on st, P's buffers set: the device form, and each chunk of the host form
static int body_mutate_device_impl(aigw_ctx* ctx, MutateParams& P, uint32_t max_len, cudaStream_t st, float* kernel_ms) {
  if (int rc = take_counters(ctx, 1, st, &P.next)) return rc;
  return timed(ctx, st, kernel_ms, [&] { CK(launch_body_mutate(P, max_len, ctx->sm_count, st)); return 0; });
}
int aigw_body_mutate_device(aigw_ctx* ctx, const aigw_body_mutation* m, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                            uint32_t max_len, uint8_t* d_out, uint64_t out_capacity, aigw_mut_result* d_results, uint64_t* d_out_used, void* stream, float* kernel_ms) {
  if (kernel_ms) *kernel_ms = 0;
  if (n == 0) return 0;
  ENTER_ON(stream);
  MutateParams P;
  if (int rc = fill_mutate_params(ctx, P, m)) return rc;
  P.bodies = d_bodies; P.offsets = d_offsets; P.lens = d_lens; P.n = n; P.out = d_out; P.out_capacity = out_capacity; P.out_bias = 0; P.results = d_results;
  P.out_used = (unsigned long long*)d_out_used;
  CK(cudaMemsetAsync(d_out_used, 0, sizeof(uint64_t), st));
  return body_mutate_device_impl(ctx, P, max_len ? max_len : 65536u, st, kernel_ms);
}
int aigw_body_mutate_host(aigw_ctx* ctx, const aigw_body_mutation* m, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n,
                          aigw_mut_batch_out* out) {
  memset(out, 0, sizeof *out);
  if (n == 0) return 0;
  ENTER();
  MutateParams P0;
  if (int rc = fill_mutate_params(ctx, P0, m)) return rc;
  uint64_t extra = 0;
  for (uint32_t k = 0; k < P0.n_keys; k++) extra += P0.keys[k].memb_len + 2;
  uint32_t max_len = 0;
  for (uint32_t i = 0; i < n; i++) if (lens[i] > max_len) max_len = lens[i];
  return chunk_pipeline(
      ctx, bodies, offsets, lens, n, 256ull << 20,
      [&](uint64_t ib, uint32_t nd) { return (ib + (uint64_t)nd * (extra + 32) + 4096 + 255) & ~255ull; }, 1,
      [&](const PipeChunk<aigw_mut_result>& k) {
        MutateParams P = P0;
        P.bodies = k.bytes; P.offsets = k.off; P.lens = k.len; P.n = k.n;
        P.out = k.out; P.out_capacity = k.out_cap; P.out_bias = k.out_bias; P.results = k.results; P.out_used = k.out_used;
        return body_mutate_device_impl(ctx, P, max_len, ctx->s_compute, nullptr);
      },
      out);
}

// ------------------------------------------------------------------ SigV4 payload hash
static int sha_common(aigw_ctx* ctx, const uint8_t* d_bytes, const uint64_t* d_off, const uint32_t* d_len, const aigw_doc_result* d_res, uint32_t n, uint8_t* d_dig, void* stream, float* kernel_ms) {
  if (kernel_ms) *kernel_ms = 0;
  if (n == 0) return 0;
  ENTER_ON(stream);
  return timed(ctx, st, kernel_ms, [&] { CK(launch_sha256(d_bytes, d_off, d_len, d_res, n, d_dig, st)); return 0; });
}
int aigw_sha256_device(aigw_ctx* ctx, const uint8_t* d_bytes, const uint64_t* d_off, const uint32_t* d_len, uint32_t n, uint8_t* d_digests, void* stream, float* kernel_ms) {
  return sha_common(ctx, d_bytes, d_off, d_len, nullptr, n, d_digests, stream, kernel_ms);
}
int aigw_chat_body_sha256_device(aigw_ctx* ctx, const uint8_t* d_out, const aigw_doc_result* d_results, uint32_t n, uint8_t* d_digests, void* stream, float* kernel_ms) {
  return sha_common(ctx, d_out, nullptr, nullptr, d_results, n, d_digests, stream, kernel_ms);
}
int aigw_sha256_host(aigw_ctx* ctx, const uint8_t* bytes, const uint64_t* off, const uint32_t* len, uint32_t n, uint8_t* digests) {
  if (n == 0) return 0;
  ENTER();
  HostStage S(ctx);
  const uint8_t* d_bytes = S.span(bytes, off, len, n);
  const uint64_t* d_off = S.in(off, n);
  const uint32_t* d_len = S.in(len, n);
  uint8_t* d_digests = S.out<uint8_t>((size_t)n * 32);
  if (S.rc) return S.rc;
  if (int rc = aigw_sha256_device(ctx, d_bytes, d_off, d_len, n, d_digests, S.st, nullptr)) return rc;
  S.back(digests, d_digests, (size_t)n * 32);
  return S.wait();
}

// ------------------------------------------------------------------ CEL cost expressions
int aigw_cost_compile(aigw_ctx* ctx, const char* expr, aigw_cost_program** out) {
  *out = nullptr;
  ENTER();
  std::unique_ptr<aigw_cost_program> p(new aigw_cost_program());   // freed with its device copies unless it is handed out
  std::string err;
  const int rc = cel_compile(expr ? expr : "", p->h, err);
  if (rc) { ctx->err = std::string(rc == 1 ? "CEL expression outside the compiled subset: " : "CEL expression rejected: ") + err; return rc == 1 ? -2 : -3; }
  std::vector<CelInstr> padded(p->h.code); padded.resize(kCelMaxInstr, CelInstr{});
  if (cudaMalloc(&p->h.d_code, sizeof(CelInstr) * kCelMaxInstr) != cudaSuccess || cudaMalloc(&p->h.d_strings, p->h.strings.size() + 16) != cudaSuccess) { ctx->err = "cudaMalloc"; return (int)cudaErrorMemoryAllocation; }
  CK(cudaMemcpy(p->h.d_code, padded.data(), sizeof(CelInstr) * kCelMaxInstr, cudaMemcpyHostToDevice));
  if (!p->h.strings.empty()) CK(cudaMemcpy(p->h.d_strings, p->h.strings.data(), p->h.strings.size(), cudaMemcpyHostToDevice));
  *out = p.release();
  return 0;
}
void aigw_cost_program_free(aigw_ctx* ctx, aigw_cost_program* p) { if (!p) return; cudaSetDevice(ctx->device); delete p; }

static int cel_fill(aigw_ctx* ctx, CelLaunch& L, aigw_cost_program* const* progs, uint32_t n_progs, const char* model, const char* backend, const char* route) {
  if (n_progs > (uint32_t)kCelMaxProgs) { ctx->err = "more than 8 CEL programs per call"; return -2; }
  memset(&L.cs, 0, sizeof L.cs);
  auto put = [&](char* dst, uint32_t& len, const char* src) -> bool { const size_t l = src ? strlen(src) : 0; if (l >= (size_t)kCelStrCap) return false; if (l) memcpy(dst, src, l); len = (uint32_t)l; return true; };
  if (!put(L.cs.model, L.cs.model_len, model) || !put(L.cs.backend, L.cs.backend_len, backend) || !put(L.cs.route, L.cs.route_len, route)) { ctx->err = "model / backend / route_name longer than 255 bytes"; return -2; }
  L.n_progs = n_progs;
  for (uint32_t p = 0; p < n_progs; p++) {
    const CelProgramHost& h = progs[p]->h;
    L.code[p] = h.d_code; L.strings[p] = h.d_strings; L.result_is_int[p] = h.result_is_int;
    uint32_t bits = 0;
    for (size_t k = 0; k < h.sites.size(); k++) {   // string comparisons that do not involve the per-record model
      const CelHostSite& st = h.sites[k];
      auto str = [&](uint8_t kind, uint32_t off, uint32_t len) { return kind == 0 ? h.strings.substr(off, len) : kind == 1 ? std::string(L.cs.backend, L.cs.backend_len) : std::string(L.cs.route, L.cs.route_len); };
      if ((str(st.lk, st.loff, st.llen) == str(st.rk, st.roff, st.rlen)) != st.negate) bits |= 1u << k;
    }
    L.host_bits[p] = bits;
  }
  return 0;
}
int aigw_usage_costs_cel_device(aigw_ctx* ctx, const aigw_sse_result* d_results, uint32_t n, aigw_cost_program* const* progs, uint32_t n_progs,
                                const uint8_t* d_model_bytes, const uint32_t* d_model_off, const uint32_t* d_model_len, const char* model, const char* backend,
                                const char* route_name, uint64_t* d_costs, uint8_t* d_errs, void* stream) {
  if (n == 0 || n_progs == 0) return 0;
  ENTER_ON(stream);
  CelLaunch L;
  if (int rc = cel_fill(ctx, L, progs, n_progs, model, backend, route_name)) return rc;
  L.results = d_results; L.n = n; L.model_bytes = d_model_bytes; L.model_off = d_model_off; L.model_len = d_model_len;
  L.costs = (unsigned long long*)d_costs; L.errs = d_errs;
  CK(launch_cel(L, st));
  return 0;
}
int aigw_usage_costs_cel_host(aigw_ctx* ctx, const aigw_sse_result* results, uint32_t n, aigw_cost_program* const* progs, uint32_t n_progs,
                              const uint8_t* model_bytes, uint64_t model_bytes_len, const uint32_t* model_off, const uint32_t* model_len, const char* model,
                              const char* backend, const char* route_name, uint64_t* costs, uint8_t* errs) {
  if (n == 0 || n_progs == 0) return 0;
  ENTER();
  const size_t nout = (size_t)n * n_progs;
  const bool spans = model_off && model_len;   // a request model per record
  HostStage S(ctx);
  const aigw_sse_result* d_results = S.in(results, n);
  const uint32_t* d_model_off = spans ? S.in(model_off, n) : nullptr;
  const uint32_t* d_model_len = spans ? S.in(model_len, n) : nullptr;
  const uint8_t* d_model_bytes = spans ? S.in(model_bytes, model_bytes_len) : nullptr;
  uint64_t* d_costs = S.out<uint64_t>(nout);
  uint8_t* d_errs = S.out<uint8_t>(nout);
  if (S.rc) return S.rc;
  if (int rc = aigw_usage_costs_cel_device(ctx, d_results, n, progs, n_progs, d_model_bytes, d_model_off, d_model_len, model, backend, route_name, d_costs, d_errs, S.st)) return rc;
  S.back(costs, d_costs, nout);
  S.back(errs, d_errs, nout);
  return S.wait();
}

// ------------------------------------------------------------------ R1 + C2
static int response_usage_device_impl(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                                      aigw_sse_result* d_results, void* stream, float* kernel_ms, int embeddings) {
  ENTER_ON(stream);
  return timed(ctx, st, kernel_ms, [&] { CK(launch_response_usage(d_bodies, d_offsets, d_lens, n, d_results, st, embeddings)); return 0; });
}

int aigw_response_usage_device(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                               aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  return response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, stream, kernel_ms, 0);
}
int aigw_embeddings_response_usage_device(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                                          aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  return response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, stream, kernel_ms, 1);
}
int aigw_completions_response_usage_device(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                                           aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  return response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, stream, kernel_ms, 2);
}
int aigw_responses_response_usage_device(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                                           aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  return response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, stream, kernel_ms, 3);
}
int aigw_rerank_response_usage_device(aigw_ctx* ctx, const uint8_t* d_bodies, const uint64_t* d_offsets, const uint32_t* d_lens, uint32_t n,
                                      aigw_sse_result* d_results, void* stream, float* kernel_ms) {
  return response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, stream, kernel_ms, 4);
}

static int response_usage_host_impl(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                                    const int32_t* cost_types, uint32_t n_costs, uint64_t* costs, int embeddings) {
  if (n == 0) return 0;
  ENTER();
  HostStage S(ctx);
  const uint8_t* d_bodies = S.span(bodies, offsets, lens, n);
  const uint64_t* d_offsets = S.in(offsets, n);
  const uint32_t* d_lens = S.in(lens, n);
  aigw_sse_result* d_results = S.out<aigw_sse_result>(n);
  if (S.rc) return S.rc;
  if (int rc = response_usage_device_impl(ctx, d_bodies, d_offsets, d_lens, n, d_results, S.st, nullptr, embeddings)) return rc;   // untimed: no wait
  S.back(results, d_results, n);
  if (n_costs && costs) {
    const int32_t* d_cost_types = S.in(cost_types, n_costs);
    uint64_t* d_costs = S.out<uint64_t>((size_t)n * n_costs);
    if (S.rc) return S.rc;
    if (int rc = aigw_usage_costs_device(ctx, d_results, n, d_cost_types, n_costs, d_costs, S.st)) return rc;
    S.back(costs, d_costs, (size_t)n * n_costs);
  }
  return S.wait();
}
int aigw_response_usage_host(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                             const int32_t* cost_types, uint32_t n_costs, uint64_t* costs) {
  return response_usage_host_impl(ctx, bodies, offsets, lens, n, results, cost_types, n_costs, costs, 0);
}
int aigw_embeddings_response_usage_host(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                                        const int32_t* cost_types, uint32_t n_costs, uint64_t* costs) {
  return response_usage_host_impl(ctx, bodies, offsets, lens, n, results, cost_types, n_costs, costs, 1);
}
int aigw_completions_response_usage_host(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                                         const int32_t* cost_types, uint32_t n_costs, uint64_t* costs) {
  return response_usage_host_impl(ctx, bodies, offsets, lens, n, results, cost_types, n_costs, costs, 2);
}
int aigw_responses_response_usage_host(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                                         const int32_t* cost_types, uint32_t n_costs, uint64_t* costs) {
  return response_usage_host_impl(ctx, bodies, offsets, lens, n, results, cost_types, n_costs, costs, 3);
}
int aigw_rerank_response_usage_host(aigw_ctx* ctx, const uint8_t* bodies, const uint64_t* offsets, const uint32_t* lens, uint32_t n, aigw_sse_result* results,
                                    const int32_t* cost_types, uint32_t n_costs, uint64_t* costs) {
  return response_usage_host_impl(ctx, bodies, offsets, lens, n, results, cost_types, n_costs, costs, 4);
}

int aigw_usage_costs_device(aigw_ctx* ctx, const aigw_sse_result* d_results, uint32_t n, const int32_t* d_cost_types, uint32_t n_costs, uint64_t* d_costs, void* stream) {
  ENTER_ON(stream);
  CK(launch_usage_costs(d_results, n, d_cost_types, n_costs, (unsigned long long*)d_costs, st));
  return 0;
}

}  // extern "C"
