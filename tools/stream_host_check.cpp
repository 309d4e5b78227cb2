// Test tooling, not product: compiles the per-thread stream step functions of aigw_b200/csrc/stream_kernel.cu for the HOST
// (g++; cuda_runtime.h turns __device__ into nothing outside nvcc) so that a new stream parser can be checked against the oracle
// on a CPU-only machine before it is run on the GPU.  Protocol on stdin, one command per line:
//   open <kind> <request_model>            -> new slot
//   feed <hex bytes> <eos 0|1>             -> prints: <status> <body_kind> <carry_len> <usage: in out total cached cc reasoning mask> <model hex> <body hex>
//                                             <out_cap: the call's output range, stream_out_cap of lib.cu>
// The append step of the real pipeline (stream_append_kernel) is restated in appendbytes() below.
#define AIGW_HOST_HARNESS 1
#include <cstdio>
#include <iostream>
#include <string>
#include <vector>
#include "../aigw_b200/csrc/stream_kernel.cu"

using namespace aigw;

static std::vector<uint8_t> unhex(const std::string& h) { std::vector<uint8_t> v; for (size_t i = 0; i + 1 < h.size(); i += 2) v.push_back((uint8_t)std::stoi(h.substr(i, 2), nullptr, 16)); return v; }
static void hex(const uint8_t* p, size_t n) { if (!n) { printf("-"); return; } for (size_t i = 0; i < n; i++) printf("%02x", p[i]); }

int main() {
  g_chunk_schema = build_schema(); g_cmpl_schema = build_completion_schema(); g_o2a_resp_schema = build_resp_schema();
  g_conv_schema = build_schema_bedrock(); g_an_schema = build_an_schema(); g_rsp_schema = build_responses_schema();
  for (uint32_t i = 0; i < 256; i++) { uint32_t v = i; for (int k = 0; k < 8; k++) v = (v & 1u) ? 0xEDB88320u ^ (v >> 1) : v >> 1; g_crc_tab[i] = v; }
  StreamSlot* S = new StreamSlot();
  std::vector<uint8_t> out(1 << 22);
  std::string cmd;
  while (std::cin >> cmd) {
    if (cmd == "open") {
      // open <kind> <request_model> [<response_id> <created>]: the slot template aigw_stream_open_batch builds (lib.cu)
      int kind; std::string model, rest; std::cin >> kind >> model; if (model == "-") model.clear();
      std::getline(std::cin, rest);
      std::string rid; long long created = 0; { char buf[200] = {0}; if (sscanf(rest.c_str(), " %199s %lld", buf, &created) >= 1) rid = buf; if (rid == "-") rid.clear(); }
      memset(S, 0, sizeof *S); S->kind = (uint32_t)kind; S->active_index = -1; S->model_len = (uint32_t)model.size(); memcpy(S->model, model.data(), model.size());
      S->tool_index = kind == AIGW_STREAM_GCP_ANTHROPIC ? -1 : 0; S->created = created;
      if (kind == AIGW_STREAM_AWS_BEDROCK) { S->id_len = (uint32_t)rid.size(); memcpy(S->id, rid.data(), rid.size()); S->flags |= SF_HAVE_CREATED; }
    } else if (cmd == "feed") {
      std::string h; int eos; std::cin >> h >> eos; if (h == "-") h.clear();
      std::vector<uint8_t> in = unhex(h);
      if (S->kind == AIGW_STREAM_OPENAI_RESPONSES) {   // no carry: stream_append_kernel leaves the slot alone, the step reads the call's bytes
        aigw_chunk_result R; memset(&R, 0, sizeof R);
        StreamStep st{0, (uint32_t)in.size(), (uint32_t)eos, stream_out_cap(S->kind, in.size(), S->model_len), 0, 0};
        if (S->flags & SF_DEAD) R.status = (uint8_t)S->dead_status; else step_openai_responses(*S, st, in.data(), out.data(), R);
        printf("%d %d %u %u %u %u %u %u %u %u ", (int)R.status, (int)R.body_kind, S->end - S->beg, R.usage.input, R.usage.output, R.usage.total, R.usage.cached, R.usage.cache_creation, R.usage.reasoning, R.usage.mask);
        hex(out.data() + R.out_len, R.model_len); printf(" "); hex(out.data(), R.out_len); printf(" %u\n", st.out_cap);
        continue;
      }
      // stream_append_kernel: compact [beg, end) to the front, append the chunk
      const uint32_t keep = S->end - S->beg;
      memmove(S->buf, S->buf + S->beg, keep); S->beg = 0; S->end = keep; S->_r0 = keep;
      aigw_chunk_result R; memset(&R, 0, sizeof R);
      const uint32_t out_cap = stream_out_cap(S->kind, keep + in.size(), S->model_len);
      if (keep + in.size() > kStreamCarryCap) { printf("4 0 0 0 0 0 0 0 0 0 - - %u\n", out_cap); continue; }
      memcpy(S->buf + keep, in.data(), in.size()); S->end = keep + (uint32_t)in.size();
      memset(S->buf + S->end, 0, std::min<size_t>(16, kStreamCarryCap - S->end));
      StreamStep st{0, (uint32_t)in.size(), (uint32_t)eos, out_cap, 0, 0};
      if (S->flags & SF_DEAD) { R.status = (uint8_t)S->dead_status; }
      else switch (S->kind) {
        case AIGW_STREAM_OPENAI: step_openai(*S, st, out.data(), R); break;
        case AIGW_STREAM_AWS_BEDROCK: step_bedrock(*S, st, out.data(), R); break;
        case AIGW_STREAM_GCP_ANTHROPIC: step_anthropic(*S, st, out.data(), R); break;
        case AIGW_STREAM_GCP_GEMINI: step_gemini(*S, st, out.data(), R); break;
        case AIGW_STREAM_GCP_GEMINI_BUFFERED: step_gemini_buffered(*S, st, out.data(), R); break;
        case AIGW_STREAM_AWS_ANTHROPIC: step_aws_anthropic(*S, st, out.data(), R); break;
        case AIGW_STREAM_OPENAI_COMPLETIONS: step_openai(*S, st, out.data(), R, true); break;
        case AIGW_STREAM_MESSAGES_OPENAI: step_messages_openai(*S, st, out.data(), R); break;
        case AIGW_STREAM_MESSAGES_OPENAI_BUFFERED: step_messages_openai_buffered(*S, st, out.data(), R); break;
        case AIGW_STREAM_MESSAGES_AWS_ANTHROPIC: step_messages_aws_anthropic(*S, st, out.data(), R); break;
        case AIGW_STREAM_ANTHROPIC: step_anthropic_native(*S, st, out.data(), R); break;
        default: R.status = AIGW_DECLINED;
      }
      R.carry_len = S->end - S->beg;
      printf("%d %d %u %u %u %u %u %u %u %u ", (int)R.status, (int)R.body_kind, R.carry_len, R.usage.input, R.usage.output, R.usage.total, R.usage.cached, R.usage.cache_creation, R.usage.reasoning, R.usage.mask);
      hex(out.data() + R.out_len, R.model_len); printf(" "); hex(out.data(), R.out_len); printf(" %u\n", out_cap);
    }
  }
  return 0;
}
