// Per-thread, table-driven typed JSON walk (device).  One thread validates one JSON text against a
// schema table the way Go's json.Unmarshal validates it against a struct type (unknown keys
// skipped after a syntax check, `null` accepted for every field, duplicate keys decode again) and
// captures a few scalar fields.  Schemas are data: a new response type is a new table.
//
// Decoder behaviour restated (github.com/bytedance/sonic v1.15.1 defaults, listed in DESIGN.md):
// control characters inside strings are accepted, UTF-8 is not validated, escapes must be
// well-formed, numbers follow RFC 8259, integer fields reject fraction/exponent/overflow.
#pragma once
#include <stdint.h>

namespace aigw { namespace tj {

enum Kind : uint8_t { K_ANY = 0, K_STR, K_INT, K_FLOAT, K_BOOL, K_OBJ, K_ARR, K_CREATED, K_B64, K_STROBJ /* string, or the object node in `elem` */,
                      K_MAP /* map[string]T: an object with arbitrary keys whose values are all of node `elem` */,
                      // the kinds below are walked only by walk<CAP, true> (the Responses API schema) and K_F64 only by walk<CAP, EXT, true>
                      // (the rerank schema); the other schemas compile without them
                      K_UNION /* tagged union: an object whose first top-level "type" string picks the variant node from the tag table
                                 fields[f0, f0+nf) (key = tag); null, a non-object, an unknown tag or a missing / non-string "type" fail */,
                      K_STRARR /* a string, or the array node in `elem`; anything else, null included, fails */,
                      K_DECLINE /* a member the schema knows but does not restate: any value sets `weird` */,
                      K_PCREATED /* *JSONUNIXTime: null is nil, anything else as K_CREATED */,
                      K_F32 /* float32: a number; an exponent or more than 38 integer digits (range not restated) sets `weird` */,
                      K_F64 /* float64: a number; an exponent or more than 308 integer digits (overflow not restated) sets `weird`.  With a
                               capture, ints[cap] = uint32(float64(text)) (f64_trunc_u32; `weird` when that is not defined) */ };

struct Field { uint16_t koff; uint8_t klen; uint8_t node; };  // key bytes at keys[koff..koff+klen)
struct Node { uint8_t kind; uint8_t cap; uint8_t f0; uint8_t nf; uint8_t elem; };

// Capture sink: up to 8 integer captures (uint32 wrap), 2 span captures, "object present" bits.
template <int NSPANS>
struct CaptureT {
  uint32_t ints[8];
  uint32_t int_set;        // bit i: ints[i] was written
  uint32_t obj_seen;       // bit cap: a non-null object with that capture id was decoded
  uint32_t span_off[NSPANS], span_len[NSPANS];
  uint32_t span_set;       // bit i
  uint32_t span_esc;       // bit i: the captured string contains a backslash
  uint32_t weird;          // escape in a key, duplicate known key, nesting too deep (typed or skipped): caller must not trust the result
  uint32_t big;            // a captured integer does not fit in 31 bits
};
using Capture = CaptureT<2>;

__device__ __forceinline__ bool ws(uint32_t c) { return c == ' ' || c == '\n' || c == '\r' || c == '\t'; }
__device__ __forceinline__ bool dig(uint32_t c) { return c - '0' < 10u; }
__device__ __forceinline__ bool delim(uint32_t c) { return ws(c) || c == ',' || c == '}' || c == ']'; }
__device__ __forceinline__ int hexv(uint32_t c) { if (c - '0' < 10u) return c - '0'; c |= 0x20; if (c - 'a' < 6u) return c - 'a' + 10; return -1; }

// string at p[i] == '"'.  Returns index after the closing quote, or -1.  esc: saw a backslash.
__device__ inline int scan_string(const uint8_t* p, int i, int n, bool& esc) {
  i++;
  while (i < n) {
    uint32_t c = p[i];
    if (c == '"') return i + 1;
    if (c == '\\') {
      esc = true;
      if (i + 1 >= n) return -1;
      uint32_t e = p[i + 1];
      if (e == 'u') { if (i + 6 > n) return -1; for (int k = 2; k < 6; k++) if (hexv(p[i + k]) < 0) return -1; i += 6; continue; }
      if (!(e == '"' || e == '\\' || e == '/' || e == 'b' || e == 'f' || e == 'n' || e == 'r' || e == 't')) return -1;
      i += 2; continue;
    }
    i++;
  }
  return -1;
}
// RFC 8259 number at p[i]; returns end index or -1; is_int: no fraction/exponent
__device__ inline int scan_number(const uint8_t* p, int i, int n, bool& is_int, int& int_end) {
  if (i < n && p[i] == '-') i++;
  if (i >= n) return -1;
  if (p[i] == '0') i++;
  else if (p[i] >= '1' && p[i] <= '9') { while (i < n && dig(p[i])) i++; }
  else return -1;
  int_end = i; is_int = true;
  if (i < n && p[i] == '.') { is_int = false; i++; if (i >= n || !dig(p[i])) return -1; while (i < n && dig(p[i])) i++; }
  if (i < n && (p[i] == 'e' || p[i] == 'E')) { is_int = false; i++; if (i < n && (p[i] == '+' || p[i] == '-')) i++; if (i >= n || !dig(p[i])) return -1; while (i < n && dig(p[i])) i++; }
  return i;
}
__device__ inline bool lit(const uint8_t* p, int i, int n, const char* w, int l) { if (i + l > n) return false; for (int k = 0; k < l; k++) if (p[i + k] != (uint8_t)w[k]) return false; return true; }
// strconv.ParseInt(s, 10, 64) on -?digits: false on overflow.  out = low 32 bits (Go uint32(int) conversion).
__device__ inline bool parse_i64(const uint8_t* p, int b, int e, uint32_t& low32, bool* big = nullptr) {
  bool neg = p[b] == '-'; if (neg) b++;
  unsigned long long v = 0;
  for (int i = b; i < e; i++) {
    unsigned d = p[i] - '0';
    if (v > (0xFFFFFFFFFFFFFFFFull - d) / 10ull) return false;
    v = v * 10ull + d;
  }
  if (neg) { if (v > 0x8000000000000000ull) return false; low32 = (uint32_t)(0ull - v); }
  else { if (v > 0x7FFFFFFFFFFFFFFFull) return false; low32 = (uint32_t)v; }
  if (big) *big = neg ? v != 0 : (v >> 31) != 0;
  return true;
}

// uint32(float64(text)) for a number without exponent whose integer digits are p[b, ie) (b after an optional '-') and whose
// fraction digits, if any, are p[ie + 1, j).  Go truncates toward zero after rounding the text to the nearest float64, so the result
// is the integer part I, or I + 1 when the text rounds up to it.  That happens iff the fraction is >= 1 - 2^-q: the float64s just
// below I + 1 are 2^(floor(log2 I) - 52) apart (2^-53 below 1), q = 53 - floor(log2 I) (54 for I = 0), and the tie goes to I + 1,
// whose mantissa is even.  1 - 2^-q has q decimals, so the test reads the first q fraction digits F (zero-padded): F >= 10^q - 5^q,
// i.e. the nines' complement of F is below 5^q < 10^38.  false: the rounded value lies outside (-1, 2^32), where Go's conversion is
// implementation-defined.
__device__ inline bool f64_trunc_u32(const uint8_t* p, int i, int ie, int j, uint32_t& out) {
  const bool neg = p[i] == '-';
  const int b = i + (neg ? 1 : 0);
  if (ie - b > 10) return false;
  unsigned long long I = 0;
  for (int k = b; k < ie; k++) I = I * 10ull + (p[k] - '0');
  if (I > 0xffffffffull || (neg && I)) return false;
  if (ie < j) {
    int fl = 0;   // floor(log2 I); a loop rather than __clzll so that the host build of the walker compiles too
    for (unsigned long long t = I; t > 1; t >>= 1) fl++;
    const int f0 = ie + 1, q = I ? 53 - fl : 54;
    bool up = true;
    unsigned __int128 c = 0, five = 1;
    for (int k = 0; k < q; k++) {
      const uint32_t cd = 9u - (f0 + k < j ? (uint32_t)(p[f0 + k] - '0') : 0u);
      if (k < q - 38) { if (cd) { up = false; break; } }
      else c = c * 10u + cd;
      five *= 5u;
    }
    if (up && c < five) {
      if (neg || I == 0xffffffffull) return false;   // -1.0, 2^32
      I++;
    }
  }
  out = (uint32_t)I;
  return true;
}

// Untyped value: syntax only.  Returns end index, -1 on a syntax error, or -2 when a container opens 65 deep inside the value (the
// isobj bitmask holds 64 levels).  -2 is not a verdict on the text: the decoder accepts deeper nesting, so callers decline.
__device__ inline int skip_any(const uint8_t* p, int i, int n) {
  uint64_t isobj = 0; int depth = 0;
  // state machine identical in spirit to validate_tokens, but byte driven
  for (;;) {
    while (i < n && ws(p[i])) i++;
    if (i >= n) return -1;
    uint32_t c = p[i];
    bool value_done = false;
    if (c == '"') { bool e = false; i = scan_string(p, i, n, e); if (i < 0) return -1; value_done = true; }
    else if (c == '{') {
      if (depth >= 64) return -2;
      i++; while (i < n && ws(p[i])) i++;
      if (i < n && p[i] == '}') { i++; value_done = true; }
      else {
        isobj |= 1ull << depth; depth++;
        // key
        if (i >= n || p[i] != '"') return -1;
        bool e = false; i = scan_string(p, i, n, e); if (i < 0) return -1;
        while (i < n && ws(p[i])) i++;
        if (i >= n || p[i] != ':') return -1;
        i++; continue;
      }
    } else if (c == '[') {
      if (depth >= 64) return -2;
      i++; while (i < n && ws(p[i])) i++;
      if (i < n && p[i] == ']') { i++; value_done = true; }
      else { isobj &= ~(1ull << depth); depth++; continue; }
    } else if (c == 't') { if (!lit(p, i, n, "true", 4)) return -1; i += 4; value_done = true; }
    else if (c == 'f') { if (!lit(p, i, n, "false", 5)) return -1; i += 5; value_done = true; }
    else if (c == 'n') { if (!lit(p, i, n, "null", 4)) return -1; i += 4; value_done = true; }
    else { bool ii; int ie; i = scan_number(p, i, n, ii, ie); if (i < 0) return -1; value_done = true; }
    // after a value: close containers / next member
    while (value_done) {
      if (depth == 0) return i;
      while (i < n && ws(p[i])) i++;
      if (i >= n) return -1;
      uint32_t d = p[i];
      bool obj = (isobj >> (depth - 1)) & 1;
      if (d == ',') {
        i++;
        if (obj) {
          while (i < n && ws(p[i])) i++;
          if (i >= n || p[i] != '"') return -1;
          bool e = false; i = scan_string(p, i, n, e); if (i < 0) return -1;
          while (i < n && ws(p[i])) i++;
          if (i >= n || p[i] != ':') return -1;
          i++;
        }
        value_done = false;
      } else if ((d == '}' && obj) || (d == ']' && !obj)) { i++; depth--; }
      else return -1;
    }
  }
}

// gjson.GetBytes(data, "type") on the object at p[i] == '{': the first top-level "type" member.  1: a string, its contents at
// p[ts, ts+tl); 0: absent or not a string; -1: syntax error before it; -2: an escaped member name before it, an escaped tag, or a
// member before it nested beyond skip_any's 64 levels.
__device__ inline int union_tag(const uint8_t* p, int i, int n, int& ts, int& tl) {
  i++;
  for (;;) {
    while (i < n && ws(p[i])) i++;
    if (i >= n) return -1;
    if (p[i] == '}') return 0;
    if (p[i] == ',') { i++; while (i < n && ws(p[i])) i++; }
    if (i >= n || p[i] != '"') return -1;
    bool e = false; const int j = scan_string(p, i, n, e); if (j < 0) return -1;
    if (e) return -2;
    const bool is_type = j - i == 6 && p[i + 1] == 't' && p[i + 2] == 'y' && p[i + 3] == 'p' && p[i + 4] == 'e';
    i = j; while (i < n && ws(p[i])) i++;
    if (i >= n || p[i] != ':') return -1;
    i++; while (i < n && ws(p[i])) i++;
    if (is_type) {
      if (i >= n || p[i] != '"') return 0;
      bool e2 = false; const int k = scan_string(p, i, n, e2); if (k < 0) return -1;
      if (e2) return -2;
      ts = i + 1; tl = k - i - 2; return 1;
    }
    i = skip_any(p, i, n); if (i < 0) return i;
  }
}

// Typed walk of p[0..n).  Returns true when json.Unmarshal into the schema's root type would succeed.  EXT: the schema uses the
// kinds from K_UNION to K_F32.  F64: the schema uses K_F64 (a separate flag: its exact conversion would otherwise enlarge the
// stack frame of every EXT walk).
template <class CAP, bool EXT = false, bool F64 = false>
__device__ inline bool walk(const uint8_t* p, int n, const Node* nodes, const Field* fields, const char* keys, int root, CAP& cap, bool allow_trailing = false) {
  const int MAXD = 12;
  uint8_t st_node[MAXD]; uint32_t st_seen[MAXD];
  int sp = 0;
  int node = root;
  int i = 0;
  for (;;) {
    // ---- a value of type `node` starts here
    while (i < n && ws(p[i])) i++;
    if (i >= n) return false;
    Node nd = nodes[node];
    uint32_t c = p[i];
    if (nd.kind == K_STROBJ) { if (c == '"' || c == 'n') nd.kind = K_STR; else { node = nd.elem; nd = nodes[node]; } }
    if constexpr (EXT) {
      if (nd.kind == K_STRARR) { if (c == '"') nd.kind = K_STR; else if (c == '[') { node = nd.elem; nd = nodes[node]; } else return false; }
      if (nd.kind == K_UNION) {   // the union's UnmarshalJSON: gjson "type", then json.Unmarshal into the variant
        if (c != '{') return false;
        int ts = 0, tl = 0; const int r = union_tag(p, i, n, ts, tl);
        if (r == -2) { cap.weird = 1; return false; }
        if (r <= 0) return false;
        int v = -1;
        for (int f = 0; f < nd.nf && v < 0; f++) {
          const Field fd = fields[nd.f0 + f];
          if (fd.klen == tl) { const char* fk = keys + fd.koff; int t = 0; while (t < tl && p[ts + t] == (uint8_t)fk[t]) t++; if (t == tl) v = fd.node; }
        }
        if (v < 0) return false;   // unknown tag
        node = v; nd = nodes[node];
      }
      if (nd.kind == K_DECLINE) { cap.weird = 1; return false; }
      if (nd.kind == K_PCREATED) nd.kind = c == 'n' ? K_ANY : K_CREATED;
      if (nd.kind == K_F32) {
        nd.kind = K_FLOAT;
        bool ii; int ie; const int j = (c == '-' || dig(c)) ? scan_number(p, i, n, ii, ie) : -1;
        if (j >= 0) { bool ex = false; for (int k = ie; k < j; k++) ex |= (p[k] | 0x20) == 'e'; if (ex || ie - i - (c == '-') > 38) cap.weird = 1; }
      }
    }
    if constexpr (F64) {
      if (nd.kind == K_F64) {
        const uint8_t fc = nd.cap; nd.kind = K_FLOAT; nd.cap = 0xff;
        bool ii; int ie; const int j = (c == '-' || dig(c)) ? scan_number(p, i, n, ii, ie) : -1;
        if (j >= 0) {
          bool ex = false; for (int k = ie; k < j; k++) ex |= (p[k] | 0x20) == 'e';
          uint32_t v;
          if (ex || ie - i - (c == '-') > 308) cap.weird = 1;
          else if (fc != 0xff) { if (!f64_trunc_u32(p, i, ie, j, v)) cap.weird = 1; else { cap.ints[fc] = v; cap.int_set |= 1u << fc; } }
        }
      }
    }
    bool descend = false;
    if (nd.kind == K_ANY) {
      const int j = skip_any(p, i, n);
      if (j == -2) { cap.weird = 1; return false; }
      if (j < 0) return false;
      if (nd.cap != 0xff) { const uint32_t s = nd.cap; cap.span_off[s] = i; cap.span_len[s] = j - i; cap.span_set |= 1u << s; }   // raw value (quotes included for strings)
      i = j;
    }
    else if (c == 'n') {
      if (!lit(p, i, n, "null", 4)) return false;
      i += 4;
      if (nd.kind == K_CREATED) return false;  // JSONUNIXTime.UnmarshalJSON is called with "null" and fails
    } else switch (nd.kind) {
      case K_STR: case K_B64: {
        if (c != '"') return false;
        bool e = false; int j = scan_string(p, i, n, e); if (j < 0) return false;
        if (nd.kind == K_B64) {  // []byte: base64.StdEncoding of the decoded string
          if (e) cap.weird = 1;
          int L = j - i - 2; const uint8_t* q = p + i + 1;
          if (L % 4) return false;
          for (int k = 0; k < L; k++) { uint32_t ch = q[k]; if (ch < 0x20) cap.weird = 1; bool ok = (ch - 'A' < 26u) || (ch - 'a' < 26u) || (ch - '0' < 10u) || ch == '+' || ch == '/' || (ch == '=' && k >= L - 2); if (!ok) return false; }
          if (L >= 2 && q[L - 2] == '=' && q[L - 1] != '=') return false;
        }
        if (nd.cap != 0xff) { const uint32_t s = nd.cap; cap.span_off[s] = i + 1; cap.span_len[s] = j - i - 2; cap.span_set |= 1u << s; if (e) cap.span_esc |= 1u << s; else cap.span_esc &= ~(1u << s); }
        i = j; break;
      }
      case K_INT: case K_FLOAT: case K_CREATED: {
        if (!(c == '-' || dig(c))) return false;
        bool ii; int ie; int j = scan_number(p, i, n, ii, ie); if (j < 0) return false;
        if (j < n && !delim(p[j])) return false;
        if (nd.kind == K_INT) { if (!ii) return false; uint32_t v; bool bg = false; if (!parse_i64(p, i, j, v, &bg)) return false; if (nd.cap != 0xff) { cap.ints[nd.cap] = v; cap.int_set |= 1u << nd.cap; if (bg) cap.big = 1; } }
        else if (nd.kind == K_CREATED) {  // integer part up to '.', exponent without '.' fails ParseInt
          if (!ii && (ie >= j || p[ie] != '.')) return false;
          uint32_t v; if (!parse_i64(p, i, ie, v)) return false;
        }
        i = j; break;
      }
      case K_BOOL: {
        if (c == 't') { if (!lit(p, i, n, "true", 4)) return false; i += 4; }
        else if (c == 'f') { if (!lit(p, i, n, "false", 5)) return false; i += 5; }
        else return false;
        break;
      }
      case K_OBJ: case K_MAP: {
        if (c != '{') return false;
        if (nd.cap != 0xff) cap.obj_seen |= 1u << nd.cap;
        i++; while (i < n && ws(p[i])) i++;
        if (i < n && p[i] == '}') { i++; break; }
        if (sp >= MAXD) { cap.weird = 1; return false; }
        st_node[sp] = (uint8_t)node; st_seen[sp] = 0; sp++;
        descend = true; break;
      }
      case K_ARR: {
        if (c != '[') return false;
        i++; while (i < n && ws(p[i])) i++;
        if (i < n && p[i] == ']') { i++; break; }
        if (sp >= MAXD) { cap.weird = 1; return false; }
        st_node[sp] = (uint8_t)node; st_seen[sp] = 0; sp++;
        node = nd.elem; continue;
      }
      default: return false;
    }
    // ---- after a value (or at the first member of an object)
    for (;;) {
      if (!descend) {
        if (sp == 0) { if (allow_trailing) return true; while (i < n && ws(p[i])) i++; return i == n; }
        while (i < n && ws(p[i])) i++;
        if (i >= n) return false;
        const Node par = nodes[st_node[sp - 1]];
        uint32_t d = p[i];
        if (par.kind == K_ARR) {
          if (d == ',') { i++; node = par.elem; break; }
          if (d == ']') { i++; sp--; continue; }
          return false;
        }
        if (d == '}') { i++; sp--; continue; }
        if (d != ',') return false;
        i++; while (i < n && ws(p[i])) i++;
      }
      descend = false;
      // object member: key ':'
      if (i >= n || p[i] != '"') return false;
      bool e = false; int j = scan_string(p, i, n, e); if (j < 0) return false;
      const uint8_t* k = p + i + 1; int kl = j - i - 2;
      if (e) cap.weird = 1;
      i = j; while (i < n && ws(p[i])) i++;
      if (i >= n || p[i] != ':') return false;
      i++;
      const Node par = nodes[st_node[sp - 1]];
      int child = -1;
      for (int f = 0; f < par.nf; f++) {
        const Field fd = fields[par.f0 + f];
        if (fd.klen == kl) {
          const char* fk = keys + fd.koff; int t = 0; while (t < kl && k[t] == (uint8_t)fk[t]) t++;
          if (t == kl) {   // a repeated member decodes again; only the first 32 members of an object are tracked (EXT schemas order the captured ones first)
            child = fd.node; const uint32_t bit = (EXT && f >= 32) ? 0u : 1u << f;
            if (st_seen[sp - 1] & bit) cap.weird = 1;
            st_seen[sp - 1] |= bit; break;
          }
        }
      }
      if (par.kind == K_MAP) child = par.elem;
      node = child < 0 ? 0 /* node 0 is K_ANY by convention */ : child;
      break;
    }
  }
}

}}  // namespace aigw::tj
