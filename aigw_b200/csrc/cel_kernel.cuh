// aigw_b200 — CEL cost expressions as device bytecode (C2 / SURVEY §8f rank 2), sm_90a.
//
// Replaces llmcostcel.NewProgram / EvaluateProgram (internal/llmcostcel/cel.go:55-99) as evalCost calls them per request at
// end of stream (internal/extproc/processor_impl.go:728-751) for the typed subset that cost expressions use: the three string
// variables (== / != only), the six uint token counters, int / uint / bool / string literals, checked + - * / %, same-type
// comparisons, ! && || with CEL's error absorption, ?:, int() / uint().  aigw_cost_compile type-checks and compiles an
// expression to a small postfix program (errors are values on the stack, so `false && <error>` is false as in CEL) and runs
// the reference's own sanity evaluation; anything outside the subset is refused at compile time (-2) so that cel-go keeps
// evaluating it.  One thread evaluates one (usage record, program) pair with the same VM the host uses for the sanity run.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>
#include <vector>

#include "../../include/aigw_b200.h"

namespace aigw {

enum CelOp : uint8_t { C_END = 0, C_PUSH_IMM, C_PUSH_TOK, C_PUSH_HOSTBIT, C_STREQ_MODEL, C_ADD_I, C_SUB_I, C_MUL_I, C_DIV_I, C_MOD_I, C_NEG_I, C_ADD_U, C_SUB_U, C_MUL_U, C_DIV_U, C_MOD_U,
                       C_EQ, C_NE, C_LT_I, C_LE_I, C_GT_I, C_GE_I, C_LT_U, C_LE_U, C_GT_U, C_GE_U, C_NOT, C_AND, C_OR, C_TO_UINT, C_TO_INT, C_JMP_FALSE, C_JMP };
enum CelErr : uint8_t { CE_OK = 0, CE_INT_OVERFLOW = 1, CE_UINT_OVERFLOW = 2, CE_DIV_ZERO = 3, CE_MOD_ZERO = 4, CE_NEGATIVE = 5 };
struct CelInstr { uint8_t op, a; uint16_t tgt; uint16_t tgt2, pad; uint64_t imm; };   // 16 bytes
static_assert(sizeof(CelInstr) == 16, "instruction layout");
constexpr int kCelMaxInstr = 96, kCelMaxStack = 16, kCelMaxProgs = 8, kCelStrCap = 256;

struct CelHostSite { uint8_t lk, rk; uint32_t loff, llen, roff, rlen; bool negate; };   // string comparison not involving `model`: resolved per call
struct CelProgramHost {
  std::vector<CelInstr> code; std::string strings; std::vector<CelHostSite> sites; bool result_is_int = false;
  CelInstr* d_code = nullptr; uint8_t* d_strings = nullptr;
};
// 0 ok, 1 outside the subset / does not type-check, 2 the reference's NewProgram would refuse it
int cel_compile(const char* expr, CelProgramHost& out, std::string& err);

struct CelStrings { char backend[kCelStrCap], route[kCelStrCap], model[kCelStrCap]; uint32_t backend_len, route_len, model_len; };
// the one VM: host (sanity evaluation) and device
__host__ __device__ inline uint8_t cel_run(const CelInstr* code, const uint8_t* strings, const uint32_t tok[6], const uint8_t* model, uint32_t model_len,
                                            const CelStrings* cs, uint32_t host_bits, bool result_is_int, uint64_t* out) {
  uint64_t st[kCelMaxStack]; uint8_t se[kCelMaxStack]; int sp = 0;
  for (int pc = 0; pc < kCelMaxInstr; pc++) {
    const CelInstr in = code[pc];
    switch (in.op) {
      case C_END: {
        const uint64_t v = st[0]; const uint8_t e = se[0];
        if (e) { *out = 0; return e; }
        if (result_is_int && (long long)v < 0) { *out = 0; return CE_NEGATIVE; }
        *out = v; return CE_OK;
      }
      case C_PUSH_IMM: st[sp] = in.imm; se[sp] = 0; sp++; break;
      case C_PUSH_TOK: st[sp] = tok[in.a]; se[sp] = 0; sp++; break;
      case C_PUSH_HOSTBIT: st[sp] = (host_bits >> in.a) & 1u; se[sp] = 0; sp++; break;
      case C_STREQ_MODEL: {   // a: 0 literal, 1 backend, 2 route; tgt: 1 = negate
        const uint8_t* p; uint32_t l;
        if (in.a == 0) { p = strings + (uint32_t)(in.imm >> 32); l = (uint32_t)in.imm; } else if (in.a == 1) { p = (const uint8_t*)cs->backend; l = cs->backend_len; } else { p = (const uint8_t*)cs->route; l = cs->route_len; }
        bool eq = l == model_len;
        for (uint32_t i = 0; eq && i < l; i++) eq = p[i] == model[i];
        st[sp] = (eq ? 1u : 0u) ^ in.tgt; se[sp] = 0; sp++; break;
      }
      case C_NOT: if (!se[sp - 1]) st[sp - 1] = !st[sp - 1]; break;
      case C_NEG_I: if (!se[sp - 1]) { if ((long long)st[sp - 1] == (long long)0x8000000000000000ull) se[sp - 1] = CE_INT_OVERFLOW; else st[sp - 1] = 0ull - st[sp - 1]; } break;
      case C_TO_UINT: if (!se[sp - 1] && (long long)st[sp - 1] < 0) se[sp - 1] = CE_UINT_OVERFLOW; break;
      case C_TO_INT: if (!se[sp - 1] && st[sp - 1] > 0x7fffffffffffffffull) se[sp - 1] = CE_INT_OVERFLOW; break;
      case C_AND: case C_OR: {
        const uint64_t a = st[sp - 2], b = st[sp - 1]; const uint8_t ea = se[sp - 2], eb = se[sp - 1]; sp--;
        const uint64_t dom = in.op == C_AND ? 0u : 1u;   // the absorbing value
        if ((!ea && a == dom) || (!eb && b == dom)) { st[sp - 1] = dom; se[sp - 1] = 0; }
        else if (ea || eb) { se[sp - 1] = ea ? ea : eb; }
        else { st[sp - 1] = 1u - dom; se[sp - 1] = 0; }
        break;
      }
      case C_JMP_FALSE: {   // tgt = else branch, tgt2 = end of the conditional (taken with the error on the stack when the condition failed)
        const uint64_t c = st[sp - 1]; const uint8_t e = se[sp - 1];
        if (e) { pc = (int)in.tgt2 - 1; break; }   // the error value stays as the conditional's result
        sp--;
        if (!c) pc = (int)in.tgt - 1;
        break;
      }
      case C_JMP: pc = (int)in.tgt - 1; break;
      default: {   // binary arithmetic / comparison
        const uint64_t a = st[sp - 2], b = st[sp - 1]; const uint8_t ea = se[sp - 2], eb = se[sp - 1]; sp--;
        uint64_t r = 0; uint8_t e = ea ? ea : eb;
        if (!e) {
          const long long x = (long long)a, y = (long long)b;
          switch (in.op) {
            case C_ADD_U: if (a > ~0ull - b) e = CE_UINT_OVERFLOW; else r = a + b; break;
            case C_SUB_U: if (a < b) e = CE_UINT_OVERFLOW; else r = a - b; break;
            case C_MUL_U: if (b && a > ~0ull / b) e = CE_UINT_OVERFLOW; else r = a * b; break;
            case C_DIV_U: if (!b) e = CE_DIV_ZERO; else r = a / b; break;
            case C_MOD_U: if (!b) e = CE_MOD_ZERO; else r = a % b; break;
            case C_ADD_I: { const unsigned long long z = a + b; if (((x >= 0) == (y >= 0)) && (((long long)z >= 0) != (x >= 0))) e = CE_INT_OVERFLOW; else r = z; break; }
            case C_SUB_I: { const unsigned long long z = a - b; if (((x >= 0) != (y >= 0)) && (((long long)z >= 0) != (x >= 0))) e = CE_INT_OVERFLOW; else r = z; break; }
            case C_MUL_I: {
              if (x == 0 || y == 0) { r = 0; break; }
              if ((x == -1 && y == (long long)0x8000000000000000ull) || (y == -1 && x == (long long)0x8000000000000000ull)) { e = CE_INT_OVERFLOW; break; }
              const long long z = (long long)(a * b);
              if (z / y != x) e = CE_INT_OVERFLOW; else r = (uint64_t)z;
              break;
            }
            case C_DIV_I: if (!y) e = CE_DIV_ZERO; else if (x == (long long)0x8000000000000000ull && y == -1) e = CE_INT_OVERFLOW; else r = (uint64_t)(x / y); break;
            case C_MOD_I: if (!y) e = CE_MOD_ZERO; else if (x == (long long)0x8000000000000000ull && y == -1) e = CE_INT_OVERFLOW; else r = (uint64_t)(x % y); break;
            case C_EQ: r = a == b; break; case C_NE: r = a != b; break;
            case C_LT_I: r = x < y; break; case C_LE_I: r = x <= y; break; case C_GT_I: r = x > y; break; case C_GE_I: r = x >= y; break;
            case C_LT_U: r = a < b; break; case C_LE_U: r = a <= b; break; case C_GT_U: r = a > b; break; case C_GE_U: r = a >= b; break;
            default: break;
          }
        }
        st[sp - 1] = r; se[sp - 1] = e;
        break;
      }
    }
  }
  *out = 0; return CE_INT_OVERFLOW;   // unreachable for compiled programs (they end with C_END)
}

struct CelLaunch {
  const aigw_sse_result* results; uint32_t n; uint32_t n_progs;
  const CelInstr* code[kCelMaxProgs]; const uint8_t* strings[kCelMaxProgs]; uint32_t host_bits[kCelMaxProgs]; uint8_t result_is_int[kCelMaxProgs];
  const uint8_t* model_bytes; const uint32_t* model_off; const uint32_t* model_len;   // per record, or NULL: cs.model for every record
  CelStrings cs;
  unsigned long long* costs; uint8_t* errs;
};
cudaError_t launch_cel(const CelLaunch& L, cudaStream_t st);

}  // namespace aigw
