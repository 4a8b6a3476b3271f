// Device ingest core: raw object JSON -> the columnar batch (program.h GkBatch), with no host parse.
//
// Reference path being replaced: the audit manager decodes every listed / spilled object from JSON into an Unstructured
// (pkg/audit/manager.go:540-551,687-695), and Matcher.Match re-unmarshals it once per constraint (pkg/target/matcher.go:73-93).
// Here ONE GPU thread per object
//   1. gk_tape_build : tokenises the object's JSON into a flat "tape" (one 64-bit entry per value / key, containers carry the
//                      index of the entry after them, so a sub-tree is skipped in O(1));
//   2. gk_ingest_obj : walks the tape along the schema's extraction program -- header fields, then a depth-first pass over the
//                      scope tree (`spec.containers[_]`, `...ports[_]`) that evaluates every feature column of a row.  It runs
//                      twice per chunk: a COUNT pass (rows per scope, bytes per byte-column), a device scan, a WRITE pass.
// Closure kinds (lower.hpp XK): Path / Elem / Key / Count are computed natively; Lut closures (a pure function of leaf
// values: canonify_cpu(limits.cpu), re_match(p, s), split(image, ":")[n] ...) hash the RAW bytes of their leaf arguments and
// look the result up in a device hash table that the host fills once per distinct argument tuple (the miss list).
//
// Written once as host/device inline code: kernels.cu runs it on the GPU (the product path); tests/_hostemu compiles the same
// functions for the CPU-only tests.  Nothing in the product library calls it on the host.
#pragma once
#include "program.h"
#include "vm_core.h"
typedef unsigned long long gk_u64;

// ---------------------------------------------------------------------------------------------- tape
enum { GK_T_END = 0, GK_T_OBJ = 1, GK_T_ARR = 2, GK_T_STR = 3, GK_T_KEY = 4, GK_T_NUM = 5, GK_T_TRUE = 6, GK_T_FALSE = 7, GK_T_NULL = 8 };
// scalar entry  : type[3:0] | esc[4] | len[31:5] | byte offset[63:32]   (strings: offset / len of the bytes BETWEEN the quotes)
// container     : type[3:0] | count[31:4]        | next[63:32]          (count: elements / members; next: entry index after it)
// A container's children are followed by one GK_T_END entry in scalar format holding the container's own byte span
// (offset of its opening bracket, length up to and including the closing one): children = [node + 1, next - 1).
#define GK_TAPE_MAX_DEPTH 64
#define GK_TAPE_LEN_MAX ((1u << 27) - 1u)

GK_HD uint32_t gk_te_type(gk_u64 e) { return (uint32_t)e & 15u; }
GK_HD uint32_t gk_te_esc(gk_u64 e) { return ((uint32_t)e >> 4) & 1u; }
GK_HD uint32_t gk_te_len(gk_u64 e) { return (uint32_t)e >> 5; }
GK_HD uint32_t gk_te_off(gk_u64 e) { return (uint32_t)(e >> 32); }
GK_HD uint32_t gk_te_count(gk_u64 e) { return (uint32_t)e >> 4; }
GK_HD uint32_t gk_te_next(gk_u64 e) { return (uint32_t)(e >> 32); }
GK_HD uint32_t gk_te_end(gk_u64 e) { return (uint32_t)(e >> 32) - 1u; }   // index of the container's GK_T_END entry
GK_HD gk_u64 gk_te_scalar(uint32_t type, uint32_t esc, uint32_t off, uint32_t len) {
  return (gk_u64)(type | (esc << 4) | (len << 5)) | ((gk_u64)off << 32);
}
GK_HD gk_u64 gk_te_container(uint32_t type, uint32_t count, uint32_t next) { return (gk_u64)(type | (count << 4)) | ((gk_u64)next << 32); }
GK_HD uint32_t gk_tape_capacity(gk_u64 json_len) { return (uint32_t)(json_len / 2u) + 4u; }   // a token needs >= 2 bytes (bar the root)

// status of one object after tokenising + header checks
enum { GK_ING_OK = 0, GK_ING_BAD_JSON = 1, GK_ING_NOT_OBJECT = 2, GK_ING_NO_KIND = 3, GK_ING_TOO_DEEP = 4, GK_ING_NULL = 5, GK_ING_TOO_LONG = 6 };

GK_HD bool gk_is_ws(uint32_t c) { return c == ' ' || c == '\n' || c == '\t' || c == '\r'; }
GK_HD bool gk_is_digit(uint32_t c) { return c >= '0' && c <= '9'; }
GK_HD int gk_hexval(uint32_t c) {
  if (c >= '0' && c <= '9') return (int)(c - '0');
  if (c >= 'a' && c <= 'f') return (int)(c - 'a' + 10);
  if (c >= 'A' && c <= 'F') return (int)(c - 'A' + 10);
  return -1;
}

// String scan, one aligned 64-bit word a step: looks for '"' or '\\' from byte p on.  The bytes of the word that lie before p are
// forced to 0xff (neither character).  The zero-byte test (v - 0x01..) & ~v & 0x80.. can only flag a wrong byte ABOVE a true hit,
// so the lowest flag is exact.  The word may reach outside [p, n): it holds at least one byte of the string, an aligned word never
// straddles a page, and hits at or past n are cut off.
// *hit: a '"' or '\\' at the returned index (< n); otherwise the returned index is where the next step starts (n: the string ran
// to the end of the text).
GK_HD uint32_t gk_scan_step(const uint8_t* js, uint32_t p, uint32_t n, bool* hit) {
  const uint32_t mis = (uint32_t)(reinterpret_cast<size_t>(js + p) & 7u);
  const gk_u64 w = *reinterpret_cast<const gk_u64*>(js + p - mis) | (mis ? ((1ull << (8u * mis)) - 1ull) : 0ull);
  const gk_u64 a = w ^ 0x2222222222222222ull, b = w ^ 0x5c5c5c5c5c5c5c5cull;
  const gk_u64 m = (((a - 0x0101010101010101ull) & ~a) | ((b - 0x0101010101010101ull) & ~b)) & 0x8080808080808080ull;
  *hit = false;
  if (m) {
#ifdef __CUDA_ARCH__
    const uint32_t at = p - mis + (uint32_t)((__ffsll((long long)m) - 1) >> 3);
#else
    const uint32_t at = p - mis + (uint32_t)(__builtin_ctzll(m) >> 3);
#endif
    if (at < n) *hit = true;
    return at < n ? at : n;
  }
  const uint32_t next = p - mis + 8u;
  return next < n ? next : n;
}

// Tokeniser: the grammar of the host parser (csrc/val.cpp JP) -- same whitespace, same escapes, same (lenient) number syntax,
// duplicate keys allowed -- so that the device accepts exactly the documents the host flattener accepts.
//
// Shape: ONE loop, one exit (rc), no read-back of the tape (the kinds of the open containers live in a 64-bit mask).  A turn of
// the loop is either one token step or -- inside a string -- one aligned 64-bit word of the string: strings are most of the
// text, and with their scan in the loop's common path (not a loop of its own inside a branch) the threads of a warp, which
// tokenise different objects, reconverge at the end of every turn whatever the lengths of their strings.
GK_HD int gk_tape_build(const uint8_t* js, uint32_t n, gk_u64* tape, uint32_t cap, uint32_t* ntape) {
  uint32_t stack[GK_TAPE_MAX_DEPTH];   // entry index of the open containers
  uint32_t cnt[GK_TAPE_MAX_DEPTH];
  uint32_t opos[GK_TAPE_MAX_DEPTH];    // byte offset of their opening brackets
  gk_u64 objmask = 0;                  // bit d: the container open at depth d is an object
  int depth = 0;
  uint32_t p = 0, t = 0;
  // state: 0 expect value, 1 after value (expect , or close), 2 expect key or '}' (just after '{'), 3 expect key (after ,)
  int state = 0;
  int rc = -1;
  bool in_str = false;                 // between the quotes of a string that started at byte s
  uint32_t s = 0, esc = 0;
  *ntape = 0;
  // (A warp vote at the head of the loop -- every thread of the warp taking its turns together -- measured slower than none:
  // the threads diverge INSIDE a turn, between the alternatives of the token step.)
  while (rc < 0) {
    const bool in_obj = depth > 0 && ((objmask >> (depth - 1)) & 1ull) != 0ull;
    if (in_str) {
      bool hit;
      p = gk_scan_step(js, p, n, &hit);
      if (!hit) {
        if (p >= n) rc = GK_ING_BAD_JSON;   // unterminated string
      } else if (js[p] == '"') {
        const uint32_t len = p - s;
        ++p;
        in_str = false;
        if (len > GK_TAPE_LEN_MAX) {
          rc = GK_ING_TOO_LONG;
        } else if (state >= 2) {
          tape[t++] = gk_te_scalar(GK_T_KEY, esc, s, len);
          while (p < n && gk_is_ws(js[p])) ++p;
          if (p >= n || js[p] != ':') {
            rc = GK_ING_BAD_JSON;
          } else {
            ++p;
            ++cnt[depth - 1];
            state = 0;
          }
        } else {
          tape[t++] = gk_te_scalar(GK_T_STR, esc, s, len);
          if (depth && !in_obj) ++cnt[depth - 1];
          state = 1;
        }
      } else {   // a backslash
        esc = 1;
        ++p;
        if (p >= n) {
          rc = GK_ING_BAD_JSON;
        } else {
          const uint32_t e = js[p];
          if (e == 'u') {
            if (n - p < 5) rc = GK_ING_BAD_JSON;
            else {
              for (int i = 1; i <= 4; ++i)
                if (gk_hexval(js[p + i]) < 0) rc = GK_ING_BAD_JSON;
              p += 4;
            }
          } else if (!(e == 'n' || e == 't' || e == 'r' || e == 'b' || e == 'f' || e == '/' || e == '\\' || e == '"')) {
            rc = GK_ING_BAD_JSON;
          }
          ++p;
        }
      }
      continue;
    }
    while (p < n && gk_is_ws(js[p])) ++p;
    const uint32_t c = p < n ? (uint32_t)js[p] : 256u;
    if (state == 1) {
      if (depth == 0) {
        rc = (p == n) ? (int)GK_ING_OK : (int)GK_ING_BAD_JSON;   // trailing characters
      } else if (c == ',') {
        ++p;
        state = in_obj ? 3 : 0;
      } else if (c == (in_obj ? (uint32_t)'}' : (uint32_t)']')) {
        ++p;
        --depth;
        if (p - opos[depth] > GK_TAPE_LEN_MAX) {
          rc = GK_ING_TOO_LONG;
        } else {
          tape[t++] = gk_te_scalar(GK_T_END, 0, opos[depth], p - opos[depth]);
          tape[stack[depth]] = gk_te_container(in_obj ? GK_T_OBJ : GK_T_ARR, cnt[depth], t);
        }
      } else {
        rc = GK_ING_BAD_JSON;
      }
    } else if (c == 256u || t + 3 >= cap) {   // (the capacity cannot run out for cap = gk_tape_capacity(n))
      rc = GK_ING_BAD_JSON;
    } else if (state == 2 && c == '}') {
      ++p;
      --depth;
      tape[t++] = gk_te_scalar(GK_T_END, 0, opos[depth], p - opos[depth]);
      tape[stack[depth]] = gk_te_container(GK_T_OBJ, 0, t);
      state = 1;
    } else if (state >= 2 && c != '"') {
      rc = GK_ING_BAD_JSON;   // object key expected
    } else if (c == '"') {   // a string starts (key or value by `state`): scanned by the turns that follow
      s = ++p;
      esc = 0;
      in_str = true;
    } else if (c == '{' || c == '[') {   // state 0: a value
      if (depth >= GK_TAPE_MAX_DEPTH) {
        rc = GK_ING_TOO_DEEP;
      } else {
        if (depth && !in_obj) ++cnt[depth - 1];
        stack[depth] = t;
        cnt[depth] = 0;
        opos[depth] = p;
        if (c == '{') objmask |= 1ull << depth;
        else objmask &= ~(1ull << depth);
        ++depth;
        tape[t++] = gk_te_container(c == '{' ? GK_T_OBJ : GK_T_ARR, 0, 0);
        ++p;
        if (c == '{') {
          state = 2;
        } else {
          while (p < n && gk_is_ws(js[p])) ++p;
          if (p < n && js[p] == ']') {
            ++p;
            --depth;
            tape[t++] = gk_te_scalar(GK_T_END, 0, opos[depth], p - opos[depth]);
            tape[stack[depth]] = gk_te_container(GK_T_ARR, 0, t);
            state = 1;
          } else {
            state = 0;
          }
        }
      }
    } else {
      uint32_t type = 0, len = 0;
      if (c == 't' && n - p >= 4 && js[p + 1] == 'r' && js[p + 2] == 'u' && js[p + 3] == 'e') {
        type = GK_T_TRUE, len = 4;
      } else if (c == 'f' && n - p >= 5 && js[p + 1] == 'a' && js[p + 2] == 'l' && js[p + 3] == 's' && js[p + 4] == 'e') {
        type = GK_T_FALSE, len = 5;
      } else if (c == 'n' && n - p >= 4 && js[p + 1] == 'u' && js[p + 2] == 'l' && js[p + 3] == 'l') {
        type = GK_T_NULL, len = 4;
      } else if (c == '-' || gk_is_digit(c)) {
        // [-] digits* then, if '.', 'e' or 'E' follows, every char of [0-9.eE+-]: the span must be a decimal literal strtod takes whole
        uint32_t q = p;
        if (js[q] == '-') ++q;
        uint32_t nint = 0, nfrac = 0;
        bool ok = true;
        while (q < n && gk_is_digit(js[q])) ++q, ++nint;
        if (q < n && (js[q] == '.' || js[q] == 'e' || js[q] == 'E')) {
          if (js[q] == '.') {
            ++q;
            while (q < n && gk_is_digit(js[q])) ++q, ++nfrac;
          }
          if (nint + nfrac == 0) ok = false;
          if (ok && q < n && (js[q] == 'e' || js[q] == 'E')) {
            uint32_t r = q + 1;
            if (r < n && (js[r] == '+' || js[r] == '-')) ++r;
            uint32_t nexp = 0;
            while (r < n && gk_is_digit(js[r])) ++r, ++nexp;
            if (nexp == 0) ok = false;
            q = r;
          }
          if (ok && q < n && (gk_is_digit(js[q]) || js[q] == '.' || js[q] == 'e' || js[q] == 'E' || js[q] == '+' || js[q] == '-')) ok = false;
        } else if (nint == 0) {
          ok = false;
        }
        if (ok) type = GK_T_NUM, len = q - p;
      }
      if (type == 0) {
        rc = GK_ING_BAD_JSON;
      } else {
        tape[t++] = gk_te_scalar(type, 0, p, len);
        p += len;
        if (depth && !in_obj) ++cnt[depth - 1];
        state = 1;
      }
    }
  }
  if (rc == GK_ING_OK) *ntape = t;
  return rc;
}

// ---------------------------------------------------------------------------------------------- strings
// A JSON string as a stream of DECODED bytes (escapes resolved exactly like the host parser, surrogate pairs included).
struct GkStr {
  const uint8_t* p;
  uint32_t n;      // raw bytes left
  uint32_t pend;   // up to 3 pending UTF-8 continuation bytes, packed little end first
  uint32_t npend;
};
GK_HD GkStr gk_str_open(const uint8_t* p, uint32_t n) {
  GkStr s;
  s.p = p;
  s.n = n;
  s.pend = 0;
  s.npend = 0;
  return s;
}
GK_HD uint32_t gk_str_hex4(const uint8_t* p) {
  return ((uint32_t)gk_hexval(p[0]) << 12) | ((uint32_t)gk_hexval(p[1]) << 8) | ((uint32_t)gk_hexval(p[2]) << 4) | (uint32_t)gk_hexval(p[3]);
}
// next decoded byte, or -1 at the end
GK_HD int gk_str_next(GkStr& s) {
  if (s.npend) {
    const int b = (int)(s.pend & 0xffu);
    s.pend >>= 8;
    --s.npend;
    return b;
  }
  if (s.n == 0) return -1;
  uint32_t c = *s.p++;
  --s.n;
  if (c != '\\') return (int)c;
  c = *s.p++;
  --s.n;
  switch (c) {
    case 'n': return '\n';
    case 't': return '\t';
    case 'r': return '\r';
    case 'b': return '\b';
    case 'f': return '\f';
    case 'u': {
      uint32_t cp = gk_str_hex4(s.p);
      s.p += 4;
      s.n -= 4;
      if (cp >= 0xD800 && cp < 0xDC00 && s.n >= 6 && s.p[0] == '\\' && s.p[1] == 'u' && gk_hexval(s.p[2]) >= 0 && gk_hexval(s.p[3]) >= 0 &&
          gk_hexval(s.p[4]) >= 0 && gk_hexval(s.p[5]) >= 0) {
        const uint32_t lo = gk_str_hex4(s.p + 2);
        s.p += 6;
        s.n -= 6;
        cp = (lo >= 0xDC00 && lo < 0xE000) ? 0x10000u + ((cp - 0xD800u) << 10) + (lo - 0xDC00u) : 0xFFFDu;
      }
      if (cp < 0x80) return (int)cp;
      if (cp < 0x800) {
        s.pend = 0x80u | (cp & 0x3Fu);
        s.npend = 1;
        return (int)(0xC0u | (cp >> 6));
      }
      if (cp < 0x10000) {
        s.pend = (0x80u | ((cp >> 6) & 0x3Fu)) | ((0x80u | (cp & 0x3Fu)) << 8);
        s.npend = 2;
        return (int)(0xE0u | (cp >> 12));
      }
      s.pend = (0x80u | ((cp >> 12) & 0x3Fu)) | ((0x80u | ((cp >> 6) & 0x3Fu)) << 8) | ((0x80u | (cp & 0x3Fu)) << 16);
      s.npend = 3;
      return (int)(0xF0u | (cp >> 18));
    }
    default: return (int)c;   // '/', '\\', '"'
  }
}

// 64-bit hash of a byte string (FNV-1a, then a finaliser): keys of the device lookup tables.  0 is reserved for "empty slot".
#define GK_HASH_INIT 0xcbf29ce484222325ull
GK_HD gk_u64 gk_hash_byte(gk_u64 h, uint32_t b) { return (h ^ (gk_u64)b) * 0x100000001b3ull; }
GK_HD gk_u64 gk_hash_fin(gk_u64 h) {
  h ^= h >> 33;
  h *= 0xff51afd7ed558ccdull;
  h ^= h >> 33;
  h *= 0xc4ceb9fe1a85ec53ull;
  h ^= h >> 33;
  return h ? h : 1ull;
}
GK_HD gk_u64 gk_hash_bytes(gk_u64 h, const uint8_t* p, uint32_t n) {
  for (uint32_t i = 0; i < n; ++i) h = gk_hash_byte(h, p[i]);
  return h;
}

// ---------------------------------------------------------------------------------------------- values
// A value the extraction program handles: a tape node of the object, or a synthetic scalar (review.kind.*, review.name,
// constants of the review envelope, array indices).
struct GkXVal {
  uint32_t vt;          // GK_VT_*
  uint32_t node;        // tape index, GK_NONE for synthetic values
  const uint8_t* sp;    // synthetic string: the bytes of a JSON string body (decoded bytes unless `sesc`)
  uint32_t slen;
  uint32_t sesc;        // the synthetic string may hold escapes (a slice of an escaped apiVersion): read it through gk_x_str
  long long inum;       // synthetic number (array index)
};
GK_HD GkXVal gk_xundef() {
  GkXVal v;
  v.vt = GK_VT_UNDEF;
  v.node = GK_NONE;
  v.sp = nullptr;
  v.slen = 0;
  v.sesc = 0;
  v.inum = 0;
  return v;
}
GK_HD GkXVal gk_xsyn(uint32_t vt) {
  GkXVal v = gk_xundef();
  v.vt = vt;
  return v;
}
GK_HD GkXVal gk_xstr(const uint8_t* p, uint32_t n) {
  GkXVal v = gk_xundef();
  v.vt = GK_VT_STR;
  v.sp = p;
  v.slen = n;
  return v;
}
GK_HD GkXVal gk_xstr_esc(const uint8_t* p, uint32_t n, uint32_t esc) {
  GkXVal v = gk_xstr(p, n);
  v.sesc = esc;
  return v;
}
GK_HD uint32_t gk_vt_of_type(uint32_t t) {
  switch (t) {
    case GK_T_OBJ: return GK_VT_OBJ;
    case GK_T_ARR: return GK_VT_ARR;
    case GK_T_STR:
    case GK_T_KEY: return GK_VT_STR;
    case GK_T_NUM: return GK_VT_NUM;
    case GK_T_TRUE: return GK_VT_TRUE;
    case GK_T_FALSE: return GK_VT_FALSE;
    case GK_T_NULL: return GK_VT_NULL;
    default: return GK_VT_UNDEF;
  }
}
GK_HD GkXVal gk_xnode(const gk_u64* tape, uint32_t node) {
  GkXVal v = gk_xundef();
  v.vt = gk_vt_of_type(gk_te_type(tape[node]));
  v.node = node;
  return v;
}
GK_HD uint32_t gk_tape_skip(const gk_u64* tape, uint32_t i) {   // entry index after the value at i
  const uint32_t t = gk_te_type(tape[i]);
  return (t == GK_T_OBJ || t == GK_T_ARR) ? gk_te_next(tape[i]) : i + 1u;
}

// the object's JSON + its tape
struct GkDoc {
  const uint8_t* js;
  const gk_u64* tape;
  uint32_t ntape;
};

// does the (decoded) string entry equal the literal?
GK_HD bool gk_entry_eq(const GkDoc& d, gk_u64 e, const uint8_t* lit, uint32_t n) {
  const uint8_t* p = d.js + gk_te_off(e);
  const uint32_t len = gk_te_len(e);
  if (!gk_te_esc(e)) {
    if (len != n) return false;
    for (uint32_t i = 0; i < n; ++i)
      if (p[i] != lit[i]) return false;
    return true;
  }
  GkStr s = gk_str_open(p, len);
  for (uint32_t i = 0; i < n; ++i)
    if (gk_str_next(s) != (int)lit[i]) return false;
  return gk_str_next(s) < 0;
}
// two (decoded) string entries equal?
GK_HD bool gk_entries_eq(const GkDoc& d, gk_u64 a, gk_u64 b) {
  if (!gk_te_esc(a) && !gk_te_esc(b)) {
    const uint32_t n = gk_te_len(a);
    if (n != gk_te_len(b)) return false;
    const uint8_t *p = d.js + gk_te_off(a), *q = d.js + gk_te_off(b);
    for (uint32_t i = 0; i < n; ++i)
      if (p[i] != q[i]) return false;
    return true;
  }
  GkStr x = gk_str_open(d.js + gk_te_off(a), gk_te_len(a)), y = gk_str_open(d.js + gk_te_off(b), gk_te_len(b));
  for (;;) {
    const int cx = gk_str_next(x), cy = gk_str_next(y);
    if (cx != cy) return false;
    if (cx < 0) return true;
  }
}

// hash of a (decoded) string entry's bytes, continuing from h
GK_HD gk_u64 gk_hash_entry(const GkDoc& d, gk_u64 e, gk_u64 h) {
  if (!gk_te_esc(e)) return gk_hash_bytes(h, d.js + gk_te_off(e), gk_te_len(e));
  GkStr s = gk_str_open(d.js + gk_te_off(e), gk_te_len(e));
  for (int b; (b = gk_str_next(s)) >= 0;) h = gk_hash_byte(h, (uint32_t)b);
  return h;
}

// member lookup: the value index of key `lit` in the object at `node`, or GK_NONE.  A repeated key means its LAST value
// (json.Unmarshal into a map; the host parser keeps the later duplicate too).
GK_HD uint32_t gk_obj_find(const GkDoc& d, uint32_t node, const uint8_t* lit, uint32_t n) {
  const gk_u64 e = d.tape[node];
  if (gk_te_type(e) != GK_T_OBJ) return GK_NONE;
  const uint32_t end = gk_te_end(e);
  uint32_t found = GK_NONE;
  for (uint32_t i = node + 1u; i < end;) {
    const gk_u64 k = d.tape[i];
    if (gk_entry_eq(d, k, lit, n)) found = i + 1u;
    i = gk_tape_skip(d.tape, i + 1u);
  }
  return found;
}
GK_HD uint32_t gk_arr_at(const GkDoc& d, uint32_t node, long long ix) {
  const gk_u64 e = d.tape[node];
  if (gk_te_type(e) != GK_T_ARR || ix < 0 || (unsigned long long)ix >= gk_te_count(e)) return GK_NONE;
  uint32_t i = node + 1u;
  for (long long j = 0; j < ix; ++j) i = gk_tape_skip(d.tape, i);
  return i;
}
// is member `ki` (key entry index) of the object ending at `end` shadowed by a later member with the same key?
GK_HD bool gk_key_shadowed(const GkDoc& d, uint32_t ki, uint32_t end) {
  const gk_u64 k = d.tape[ki];
  for (uint32_t i = gk_tape_skip(d.tape, ki + 1u); i < end; i = gk_tape_skip(d.tape, i + 1u))
    if (gk_entries_eq(d, k, d.tape[i])) return true;
  return false;
}

// ---------------------------------------------------------------------------------------------- numbers
// num_key (val.hpp) of a number token: 2*floor(x) + (x is fractional), saturated at +-(2^63 - 2).
GK_HD long long gk_num_key_token(const uint8_t* p, uint32_t n) {
  const long long SAT_HI = 0x7ffffffffffffffell, SAT_LO = -0x7ffffffffffffffell;
  uint32_t i = 0;
  bool neg = false;
  if (i < n && p[i] == '-') neg = true, ++i;
  // decimal digits of the mantissa (up to 19 significant ones kept), position of the decimal point, exponent
  unsigned long long mant = 0;
  int kept = 0, dropped_int = 0;    // digits dropped from the integer part scale the value by 10 each
  bool dropped_nonzero = false, seen_nonzero = false;
  int frac_digits = 0;
  bool in_frac = false;
  for (; i < n; ++i) {
    const uint32_t c = p[i];
    if (c == '.') {
      in_frac = true;
      continue;
    }
    if (!gk_is_digit(c)) break;
    const uint32_t dgt = c - '0';
    if (dgt) seen_nonzero = true;
    if (kept < 19) {
      mant = mant * 10ull + dgt;
      if (seen_nonzero) ++kept;
      if (in_frac) ++frac_digits;
    } else {
      if (dgt) dropped_nonzero = true;
      if (!in_frac) ++dropped_int;
    }
  }
  long long ex = 0;
  if (i < n && (p[i] == 'e' || p[i] == 'E')) {
    ++i;
    bool eneg = false;
    if (i < n && (p[i] == '+' || p[i] == '-')) eneg = p[i] == '-', ++i;
    for (; i < n && gk_is_digit(p[i]); ++i)
      if (ex < 100000) ex = ex * 10 + (p[i] - '0');
    if (eneg) ex = -ex;
  }
  // value = (mant [+ tiny]) * 10^shift
  long long shift = ex - frac_digits + dropped_int;
  if (mant == 0 && !dropped_nonzero) return 0;
  unsigned long long fl = mant;
  bool frac = dropped_nonzero;
  bool huge = false;
  if (shift > 0) {
    for (long long k = 0; k < shift && !huge; ++k) {
      if (fl > 0x3fffffffffffffffull / 10ull) huge = true;
      else fl *= 10ull;
    }
  } else if (shift < 0) {
    for (long long k = 0; k < -shift; ++k) {
      if (fl == 0) {
        break;
      }
      if (fl % 10ull) frac = true;
      fl /= 10ull;
    }
    if (mant != 0 && fl == 0) frac = true;
  }
  if (huge || fl > 0x3fffffffffffffffull) return neg ? SAT_LO : SAT_HI;
  // floor of the signed value
  if (!neg) return (long long)(2ull * fl + (frac ? 1ull : 0ull));
  // x = -(fl + f), 0 <= f < 1:  floor(x) = -fl - (f > 0)
  const long long f2 = -(long long)fl - (frac ? 1 : 0);
  return 2 * f2 + (frac ? 1 : 0);
}
// canonical-integer token: "0" or [-]?[1-9][0-9]* (its text IS num_str of the value)
GK_HD bool gk_plain_int(const uint8_t* p, uint32_t n) {
  uint32_t i = 0;
  if (n && p[0] == '-') i = 1;
  if (i >= n) return false;
  if (p[i] == '0') return n == 1;
  for (uint32_t j = i; j < n; ++j)
    if (!gk_is_digit(p[j])) return false;
  return n - i <= 18;
}

// ---------------------------------------------------------------------------------------------- lookup tables
// Open-addressing table keyed by a 64-bit hash.  val: a result index / sid, GK_HT_PENDING while the host has not filled it.
#define GK_HT_PENDING 0xFFFFFFFFu
typedef struct {
  unsigned long long* keys;   // 0 = empty
  uint32_t* vals;
  uint32_t mask;              // capacity - 1
  uint32_t pad_;
} GkHtab;

GK_HD uint32_t gk_ht_find(const GkHtab& t, gk_u64 key, bool* present) {
  uint32_t i = (uint32_t)key & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe) {
    const unsigned long long k = t.keys[i];
    if (k == key) {
      *present = true;
      return t.vals[i];
    }
    if (k == 0ull) break;
    i = (i + 1u) & t.mask;
  }
  *present = false;
  return GK_HT_PENDING;
}

// one result of a Lut closure (what the encodings of a row need)
typedef struct {
  uint32_t vt;
  uint32_t sid;
  long long num;
  uint32_t head[GK_HEAD_WORDS];
} GkLutVal;

// where a missing lookup's argument lives, for the host to evaluate: (byte offset in the blob, length) of the raw token /
// sub-tree, or a synthetic scalar
enum { GK_ARG_UNDEF = 0, GK_ARG_JSON = 1, GK_ARG_INDEX = 2, GK_ARG_SYNSTR = 3 };
typedef struct {
  uint32_t kind;
  uint32_t len;
  unsigned long long off;   // GK_ARG_JSON: absolute offset in the blob; GK_ARG_INDEX: the index; GK_ARG_SYNSTR: absolute offset of a JSON string body's bytes (the host decodes any escapes)
} GkMissArg;
#define GK_LUT_MAX_ARGS 4
typedef struct {
  uint32_t col;             // closure id (extraction-program closure table)
  uint32_t slot;            // table slot claimed for it
  unsigned long long key;
  GkMissArg args[GK_LUT_MAX_ARGS];
} GkMiss;

// ---------------------------------------------------------------------------------------------- extraction program
enum { GK_X_PATH = 1, GK_X_ELEM = 2, GK_X_KEY = 3, GK_X_COUNT = 4, GK_X_LUT = 5 };
// review-envelope roots of an `input.review.<root>...` path (pkg/target/review.go:16-29; SURVEY Appendix C)
enum { GK_R_REVIEW = 0, GK_R_OBJECT = 1, GK_R_KIND = 2, GK_R_NAME = 3, GK_R_NAMESPACE = 4, GK_R_OLDOBJECT = 5, GK_R_OPERATION = 6, GK_R_UID = 7,
       GK_R_OPTIONS = 8, GK_R_RESOURCE = 9, GK_R_USERINFO = 10, GK_R_UNDEF = 11 };
typedef struct {
  uint32_t kind;        // GK_X_*
  int32_t base;         // Path / Count: closure index the value is read from; -1: the review envelope (root in `root`)
  uint32_t root;        // GK_R_* when base < 0
  uint32_t scope;       // Elem / Key: the scope whose current row is meant
  uint32_t keys_off, nkeys;   // Path: xkeys[keys_off ..]: (is_index, byte_off | index, len) triples
  uint32_t args_off, nargs;   // Lut: xargs[args_off ..]: closure indices of the leaf arguments
  unsigned long long seed;    // Lut: hash domain
  // Lut closures made of slicing string builtins only (split / trim / index / last / count over ONE leaf string) also carry a
  // native program (GK_SX_* postfix ops in xkeys): rows whose leaf has no escape sequence never touch the lookup table --
  // image names, paths and the like are as many distinct values as there are rows.
  uint32_t sx_off, sx_n;
} GkXClosure;
enum { GK_SX_LEAF = 1 /* a = argument index */, GK_SX_SPLIT = 2 /* a,b = delimiter (byte_off, len) */, GK_SX_TRIM = 3 /* a,b = cutset */,
       GK_SX_INDEX = 4 /* a = index */, GK_SX_LAST = 5, GK_SX_COUNT = 6, GK_SX_LOWER_UNUSED = 7 };
typedef struct {
  uint32_t closure;
  uint32_t scope;
  uint32_t enc;
  uint32_t bytes_slot;  // index among the byte-counted columns (GK_ENC_BYTES), GK_NONE otherwise
} GkXCol;
typedef struct {
  uint32_t gen;         // closure index of the iterated collection
  int32_t parent;
  uint32_t first_child, next_sibling;   // scope tree (GK_NONE terminated)
  uint32_t first_col, ncols;            // columns of this scope: xcol_order[first_col ..]
} GkXScope;

typedef struct {
  const GkXClosure* cl;
  const GkXCol* cols;
  const GkXScope* scopes;
  const uint32_t* col_order;   // column indices grouped by scope
  const uint32_t* xkeys;
  const uint32_t* xargs;
  const uint8_t* xbytes;       // literal key strings
  uint32_t ncl, ncols, nscopes, nbytecols;
  // string -> sid (interned constants; a miss is GK_SID_OTHER, never pending) and the Lut results
  GkHtab sid_tab;
  GkHtab lut_tab;
  const GkLutVal* lut_vals;
  uint32_t sid_true, sid_false, sid_null;   // sids of the non-string scalars (GK_SID_OTHER when no constant mentions them)
  uint32_t pad_;
  // namespace cache as a table: name hash -> row of (nsl_off, nsl_kv); names for nsname
  GkHtab ns_tab;
  const uint32_t* nsn_off;     // [nsrows + 1] bytes of each cached Namespace's metadata.name
  const uint8_t* nsn_bytes;
  // excluder patterns of the calling process (mode, byte_off, len) in xkeys / xbytes
  uint32_t excl_off, excl_n;
} GkXProg;

#define GK_SEED_STR 0x9ae16a3b2f90404full   /* hash domain of string values -> sid */
#define GK_SEED_NUM 0xc3a5c85c97cb3127ull   /* canonical integers -> sid */
#define GK_SEED_NS 0xb492b66fbe98f273ull    /* namespace names -> namespace table row */

// per-object header counters produced by the header COUNT pass, one array of n entries each (then scanned), laid out
// [counter][object]: name bytes, generateName bytes, labels, nsname bytes
#define GK_CNT_EXTRA 4

typedef struct {
  uint32_t elem;     // tape index of the row's element
  uint32_t key;      // tape index of the member's key, or (array index | GK_ROW_INDEX)
  uint32_t parent;   // row of the parent scope (an object index under the root)
  uint32_t obj;      // object index
} GkRowRec;

// per-chunk destination arrays of the WRITE pass (device pointers; offsets are chunk-relative)
typedef struct {
  uint32_t* flags;
  uint32_t* kind_sid;
  uint32_t* group_sid;
  uint32_t* name_off;
  uint8_t* name_bytes;
  uint32_t* gen_off;
  uint8_t* gen_bytes;
  uint32_t* lbl_off;
  uint32_t* lbl_kv;
  uint32_t* nsrow;
  uint32_t* nsn_off;      // nsname bytes of each object (namespaces / excludedNamespaces match on it)
  uint8_t* nsn_bytes;
  uint32_t* const* scope_off;   // [nscopes]: [parent rows + 1]
  // columns
  uint8_t* const* vt;
  uint32_t* const* sid;
  long long* const* num;
  uint32_t* const* boff;
  uint8_t* const* bytes;
  uint32_t* const* head;
  // row handles (scratch, not part of the batch): what the per-row column pass needs to find its element again -- one
  // 16-byte record per row, written with one store
  GkRowRec* const* row_rec;      // [nscopes][rows]
  // scratch: hash of (apiVersion, kind) per object, 0 for a skipped one -- the audit asks whether a batch is of one kind
  // (results are ordered by group, version, kind first: pkg/audit/manager.go:161-202)
  gk_u64* gvk;                   // may be null
} GkIngestOut;
#define GK_ROW_INDEX 0x80000000u

typedef struct {
  const uint8_t* blob;              // the chunk's JSON bytes
  const unsigned long long* ooff;   // [n + 1] byte offsets of the objects in `blob`
  unsigned long long* tape;         // scratch: object i's tape starts at tape_off(i)
  uint32_t* ntape;                  // [n]
  uint32_t* status;                 // [n] GK_ING_*
  uint32_t n;
  uint32_t source;                  // GK_SRC_* of every object of the chunk
  uint32_t* counts;                 // [GK_CNT_EXTRA * n] header counters; after the scan: exclusive prefix sums
  GkMiss* misses;                   // miss list
  uint32_t* nmiss;
  uint32_t miss_cap;
  uint32_t pad_;
} GkIngestIn;

GK_HD unsigned long long gk_tape_off(const unsigned long long* ooff, uint32_t i) { return ooff[i] / 2ull + 4ull * (unsigned long long)i; }

// ---------------------------------------------------------------------------------------------- evaluation context
struct GkXCtx {
  GkDoc doc;
  const GkXProg* xp;
  const void* in;                // GkIngestIn of the pass (miss list of the lookup tables)
  unsigned long long blob_off;   // absolute offset of doc.js in the blob
  // review envelope
  uint32_t env_ready;            // gk_x_envelope has run
  uint32_t api_node, kind_node, name_node, ns_node, meta_node;   // tape indices or GK_NONE
  const uint8_t* grp;            // group / version slices of the raw apiVersion, cut at its first decoded '/'; each holds whole
  uint32_t grp_len;              // escapes only
  const uint8_t* ver;
  uint32_t ver_len;
  uint32_t env_esc;              // apiVersion holds escapes: the slices are read decoded (gk_x_str)
  // current row of every scope on the DFS stack
  // (kept small: this context lives in per-thread local memory, and ncu showed the column pass bound by local-memory misses --
  // 4 GB of them per 1.6 M rows -- when each depth held two 32-byte values)
  uint32_t elem_node[GK_MAX_LOOP_DEPTH + 1];  // tape index of the row's element at each depth
  uint32_t key_ref[GK_MAX_LOOP_DEPTH + 1];    // tape index of the member's key, or (array index | GK_ROW_INDEX)
  uint32_t scope_at[GK_MAX_LOOP_DEPTH + 1];   // scope id at each depth
  int depth;
  // per-row memo of the path steps: memo[closure] = tape node (16 bits: a longer tape is not memoised), GK_MEMO_UNDEF or
  // GK_MEMO_EMPTY; null: no memo
  unsigned short* memo;
};
#define GK_MEMO_EMPTY 0xfffeu
#define GK_MEMO_UNDEF 0xffffu
#define GK_MEMO_MAX 256

// review envelope fields of the object (apiVersion -> group / version, kind, metadata.name / namespace): computed on first use
GK_HD void gk_x_envelope(GkXCtx& c) {
  c.env_ready = 1;
  c.api_node = gk_obj_find(c.doc, 0, reinterpret_cast<const uint8_t*>("apiVersion"), 10);
  c.kind_node = gk_obj_find(c.doc, 0, reinterpret_cast<const uint8_t*>("kind"), 4);
  c.grp = c.ver = nullptr;
  c.grp_len = c.ver_len = 0;
  c.env_esc = 0;
  if (c.api_node != GK_NONE && gk_te_type(c.doc.tape[c.api_node]) == GK_T_STR) {
    const gk_u64 e = c.doc.tape[c.api_node];
    const uint8_t* p = c.doc.js + gk_te_off(e);
    const uint32_t len = gk_te_len(e);
    uint32_t s = 0, w = 1;   // the separator: its raw offset and width ('/', or the escapes "\/" and 'u' 002F)
    if (!gk_te_esc(e)) {
      while (s < len && p[s] != '/') ++s;
    } else {
      // the tokeniser has checked every escape: a backslash is followed by one character, or by 'u' and four hex digits, inside
      // the string.  Escapes are stepped over whole, so neither slice ends inside one.
      c.env_esc = 1;
      while (s < len && p[s] != '/') {
        if (p[s] != '\\') {
          ++s;
        } else if (p[s + 1] == '/') {
          w = 2;
          break;
        } else if (p[s + 1] != 'u') {
          s += 2;
        } else if (gk_str_hex4(p + s + 2) == 0x2Fu) {
          w = 6;
          break;
        } else {
          s += 6;
        }
      }
    }
    if (s >= len) {
      c.ver = p;
      c.ver_len = len;
      c.grp = p;
      c.grp_len = 0;
    } else {
      c.grp = p;
      c.grp_len = s;
      c.ver = p + s + w;
      c.ver_len = len - s - w;
    }
  }
  c.meta_node = gk_obj_find(c.doc, 0, reinterpret_cast<const uint8_t*>("metadata"), 8);
  c.name_node = c.ns_node = GK_NONE;
  if (c.meta_node != GK_NONE && gk_te_type(c.doc.tape[c.meta_node]) == GK_T_OBJ) {
    uint32_t nm = gk_obj_find(c.doc, c.meta_node, reinterpret_cast<const uint8_t*>("name"), 4);
    uint32_t ns = gk_obj_find(c.doc, c.meta_node, reinterpret_cast<const uint8_t*>("namespace"), 9);
    if (nm != GK_NONE && (gk_te_type(c.doc.tape[nm]) != GK_T_STR || gk_te_len(c.doc.tape[nm]) == 0)) nm = GK_NONE;
    if (ns != GK_NONE && (gk_te_type(c.doc.tape[ns]) != GK_T_STR || gk_te_len(c.doc.tape[ns]) == 0)) ns = GK_NONE;
    c.name_node = nm;
    c.ns_node = ns;
  } else {
    c.meta_node = GK_NONE;
  }
}

GK_HD GkXVal gk_x_follow(const GkXCtx& c, GkXVal v, const uint32_t* keys, uint32_t nkeys) {
  for (uint32_t j = 0; j < nkeys; ++j) {
    if (v.node == GK_NONE) return gk_xundef();   // a path into a synthetic scalar
    const uint32_t* k = keys + 3u * j;
    uint32_t nx;
    const uint32_t t = gk_te_type(c.doc.tape[v.node]);
    if (t == GK_T_OBJ) {
      if (k[0]) return gk_xundef();              // numeric key into an object: object keys are strings in JSON
      nx = gk_obj_find(c.doc, v.node, c.xp->xbytes + k[1], k[2]);
    } else if (t == GK_T_ARR) {
      if (!k[0]) return gk_xundef();
      nx = gk_arr_at(c.doc, v.node, (long long)(int32_t)k[1]);
    } else {
      return gk_xundef();
    }
    if (nx == GK_NONE) return gk_xundef();
    v = gk_xnode(c.doc.tape, nx);
  }
  return v;
}

GK_HD bool gk_lit_eq(const uint8_t* a, uint32_t n, const char* b) {
  uint32_t i = 0;
  for (; i < n && b[i]; ++i)
    if (a[i] != (uint8_t)b[i]) return false;
  return i == n && !b[i];
}

// `input.review.<root>` + keys
GK_HD GkXVal gk_x_root(const GkXCtx& cc, uint32_t root, const uint32_t* keys, uint32_t nkeys) {
  GkXCtx& c = const_cast<GkXCtx&>(cc);
  if (!c.env_ready && (root == GK_R_KIND || root == GK_R_NAME || root == GK_R_NAMESPACE)) gk_x_envelope(c);
  switch (root) {
    case GK_R_REVIEW: return nkeys ? gk_xundef() : gk_xsyn(GK_VT_OBJ);
    case GK_R_OBJECT: return gk_x_follow(c, gk_xnode(c.doc.tape, 0), keys, nkeys);
    case GK_R_KIND: {
      if (nkeys == 0) return gk_xsyn(GK_VT_OBJ);
      if (nkeys > 1 || keys[0]) return gk_xundef();
      const uint8_t* k = c.xp->xbytes + keys[1];
      const uint32_t kl = keys[2];
      if (gk_lit_eq(k, kl, "kind")) return c.kind_node != GK_NONE ? gk_xnode(c.doc.tape, c.kind_node) : gk_xstr(nullptr, 0);
      if (gk_lit_eq(k, kl, "group")) return gk_xstr_esc(c.grp, c.grp_len, c.env_esc);
      if (gk_lit_eq(k, kl, "version")) return gk_xstr_esc(c.ver, c.ver_len, c.env_esc);
      return gk_xundef();
    }
    case GK_R_NAME:
    case GK_R_NAMESPACE: {
      // present only when non-empty (engine.cpp review_doc)
      const uint32_t nd = root == GK_R_NAME ? c.name_node : c.ns_node;
      if (nd == GK_NONE || nkeys) return gk_xundef();
      return gk_xnode(c.doc.tape, nd);
    }
    case GK_R_OLDOBJECT:
    case GK_R_OPTIONS: return nkeys ? gk_xundef() : gk_xsyn(GK_VT_NULL);
    case GK_R_OPERATION:
    case GK_R_UID: return nkeys ? gk_xundef() : gk_xstr(nullptr, 0);
    case GK_R_USERINFO: return nkeys ? gk_xundef() : gk_xsyn(GK_VT_OBJ);
    case GK_R_RESOURCE: {
      if (nkeys == 0) return gk_xsyn(GK_VT_OBJ);
      if (nkeys > 1 || keys[0]) return gk_xundef();
      const uint8_t* k = c.xp->xbytes + keys[1];
      const uint32_t kl = keys[2];
      if (gk_lit_eq(k, kl, "group") || gk_lit_eq(k, kl, "version") || gk_lit_eq(k, kl, "resource")) return gk_xstr(nullptr, 0);
      return gk_xundef();
    }
    default: return gk_xundef();
  }
}

GK_HD int gk_depth_of_scope(const GkXCtx& c, uint32_t scope) {
  for (int d = c.depth; d >= 1; --d)
    if (c.scope_at[d] == scope) return d;
  return 0;
}

// value of a native closure (Path / Elem / Key) for the current rows; Count and Lut are handled by the encoder
GK_HD void gk_memo_put(const GkXCtx& c, uint32_t ci, const GkXVal& v) {
  if (!c.memo || ci >= GK_MEMO_MAX) return;
  if (v.vt == GK_VT_UNDEF) c.memo[ci] = GK_MEMO_UNDEF;
  else if (v.node < GK_MEMO_EMPTY) c.memo[ci] = (unsigned short)v.node;   // (a synthetic value -- no tape node -- is recomputed)
}
GK_HD GkXVal gk_x_eval(const GkXCtx& c, uint32_t ci) {
  // walk down from the requested closure towards its leaf base, collecting the steps still to take; stop at the first step this
  // row has taken already
  uint32_t chain[16];
  int nchain = 0;
  GkXVal v = gk_xundef();
  bool have = false;
  for (;;) {
    const GkXClosure& cl = c.xp->cl[ci];
    if (cl.kind != GK_X_PATH) break;
    if (c.memo && ci < GK_MEMO_MAX && c.memo[ci] != GK_MEMO_EMPTY) {
      const uint32_t m = c.memo[ci];
      if (m != GK_MEMO_UNDEF) v = gk_xnode(c.doc.tape, m);
      have = true;
      break;
    }
    if (cl.base < 0) {   // rooted at the review envelope: gk_x_root walks the closure's own keys
      v = gk_x_root(c, cl.root, c.xp->xkeys + cl.keys_off, cl.nkeys);
      gk_memo_put(c, ci, v);
      have = true;
      break;
    }
    if (nchain >= 16) return gk_xundef();
    chain[nchain++] = ci;
    ci = (uint32_t)cl.base;
  }
  if (!have) {
    const GkXClosure& leaf = c.xp->cl[ci];
    if (leaf.kind != GK_X_ELEM && leaf.kind != GK_X_KEY) return gk_xundef();
    const int d = gk_depth_of_scope(c, leaf.scope);
    if (d == 0) return gk_xundef();
    if (leaf.kind == GK_X_ELEM) {
      v = gk_xnode(c.doc.tape, c.elem_node[d]);
    } else if (c.key_ref[d] & 0x80000000u) {   // GK_ROW_INDEX: an array index
      v = gk_xsyn(GK_VT_NUM);
      v.inum = (long long)(c.key_ref[d] & 0x7fffffffu);
    } else {
      v = gk_xnode(c.doc.tape, c.key_ref[d]);
    }
  }
  for (int j = nchain - 1; j >= 0; --j) {
    if (v.vt != GK_VT_UNDEF) {
      const GkXClosure& cl = c.xp->cl[chain[j]];
      v = gk_x_follow(c, v, c.xp->xkeys + cl.keys_off, cl.nkeys);
    }
    gk_memo_put(c, chain[j], v);
  }
  return v;
}

// ---------------------------------------------------------------------------------------------- atomics (device / host emulation)
#ifdef __CUDA_ARCH__
#define GK_CAS64(p, cmp, val) atomicCAS((unsigned long long*)(p), (unsigned long long)(cmp), (unsigned long long)(val))
#define GK_CAS32(p, cmp, val) atomicCAS((unsigned int*)(p), (unsigned int)(cmp), (unsigned int)(val))
#define GK_ADD32(p, v) atomicAdd((unsigned int*)(p), (unsigned int)(v))
#else
static inline unsigned long long gk_cas64_host(unsigned long long* p, unsigned long long cmp, unsigned long long val) {
  __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return cmp;
}
static inline unsigned int gk_cas32_host(unsigned int* p, unsigned int cmp, unsigned int val) {
  __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST);
  return cmp;
}
#define GK_CAS64(p, cmp, val) gk_cas64_host((unsigned long long*)(p), (unsigned long long)(cmp), (unsigned long long)(val))
#define GK_CAS32(p, cmp, val) gk_cas32_host((unsigned int*)(p), (unsigned int)(cmp), (unsigned int)(val))
#define GK_ADD32(p, v) __atomic_fetch_add((unsigned int*)(p), (unsigned int)(v), __ATOMIC_SEQ_CST)
#endif
#define GK_HT_LOST 0xFFFFFFFEu   /* claimed, but the miss list was full: the next pass records it */

// Lut lookup with insertion on a miss.  Returns the result index, or GK_HT_PENDING (a miss record was / will be written).
GK_HD uint32_t gk_lut_lookup(const GkXProg& xp, const GkIngestIn& in, uint32_t closure, gk_u64 key, const GkMissArg* args, uint32_t nargs) {
  const GkHtab& t = xp.lut_tab;
  uint32_t i = (uint32_t)key & t.mask;
  for (uint32_t probe = 0; probe <= t.mask; ++probe, i = (i + 1u) & t.mask) {
    unsigned long long k = t.keys[i];
    bool mine = false;
    if (k == 0ull) {
      k = GK_CAS64(&t.keys[i], 0ull, key);
      if (k == 0ull) {
        mine = true;
        k = key;
      }
    }
    if (k != key) continue;
    uint32_t v = mine ? GK_HT_LOST : t.vals[i];
    if (v == GK_HT_LOST && (mine || GK_CAS32(&t.vals[i], GK_HT_LOST, GK_HT_PENDING) == GK_HT_LOST)) {
      // this thread records the miss
      const uint32_t m = GK_ADD32(in.nmiss, 1u);
      if (m < in.miss_cap) {
        GkMiss& ms = in.misses[m];
        ms.col = closure;
        ms.slot = i;
        ms.key = key;
        for (uint32_t a = 0; a < GK_LUT_MAX_ARGS; ++a) {
          if (a < nargs) ms.args[a] = args[a];
          else ms.args[a].kind = GK_ARG_UNDEF, ms.args[a].len = 0, ms.args[a].off = 0;
        }
        t.vals[i] = GK_HT_PENDING;
      } else {
        t.vals[i] = GK_HT_LOST;
      }
      return GK_HT_PENDING;
    }
    return (v == GK_HT_LOST) ? GK_HT_PENDING : v;
  }
  return GK_HT_PENDING;   // table full: the host grows it when the load factor passes its limit, long before this
}

#define GK_CL_SIDVAL 0xFFFFFFFFu   /* pseudo closure of the miss list: "the sid of this value" (numbers not in canonical form, composites) */
#define GK_SEED_SIDVAL 0x7d1f9b3c55aa1e67ull

// ---- string access of a value (tape string or synthetic)
GK_HD GkStr gk_x_str(const GkXCtx& c, const GkXVal& v) {
  if (v.node != GK_NONE) {
    const gk_u64 e = c.doc.tape[v.node];
    return gk_str_open(c.doc.js + gk_te_off(e), gk_te_len(e));
  }
  return gk_str_open(v.sp, v.slen);   // synthetic strings are JSON string bodies: decoded bytes without backslashes, or `sesc`
}

GK_HD uint32_t gk_x_sid_exotic(const GkXCtx& c, const GkXVal& v);
// sid of a value: strings / canonical integers / true / false / null natively; numbers in another spelling (7.0, 1e3) and
// composites through the lookup table (the host canonicalises them once per distinct spelling)
GK_HD uint32_t gk_x_sid(const GkXCtx& c, const GkXVal& v) {
  const GkXProg& xp = *c.xp;
  switch (v.vt) {
    case GK_VT_UNDEF: return GK_SID_UNDEF;
    case GK_VT_TRUE: return xp.sid_true;
    case GK_VT_FALSE: return xp.sid_false;
    case GK_VT_NULL: return xp.sid_null;
    case GK_VT_STR: {
      GkStr s = gk_x_str(c, v);
      gk_u64 h = GK_SEED_STR;
      for (int b; (b = gk_str_next(s)) >= 0;) h = gk_hash_byte(h, (uint32_t)b);
      bool present;
      const uint32_t sid = gk_ht_find(xp.sid_tab, gk_hash_fin(h), &present);
      return present ? sid : GK_SID_OTHER;
    }
    case GK_VT_NUM: {
      if (v.node == GK_NONE) {   // an array index
        uint8_t buf[24];
        uint32_t n = 0;
        long long x = v.inum;
        if (x == 0) buf[n++] = '0';
        uint8_t tmp[24];
        uint32_t m = 0;
        while (x > 0) tmp[m++] = (uint8_t)('0' + x % 10), x /= 10;
        while (m) buf[n++] = tmp[--m];
        bool present;
        const uint32_t sid = gk_ht_find(xp.sid_tab, gk_hash_fin(gk_hash_bytes(GK_SEED_NUM, buf, n)), &present);
        return present ? sid : GK_SID_OTHER;
      }
      const gk_u64 e = c.doc.tape[v.node];
      const uint8_t* p = c.doc.js + gk_te_off(e);
      const uint32_t n = gk_te_len(e);
      if (!gk_plain_int(p, n)) return gk_x_sid_exotic(c, v);
      bool present;
      const uint32_t sid = gk_ht_find(xp.sid_tab, gk_hash_fin(gk_hash_bytes(GK_SEED_NUM, p, n)), &present);
      return present ? sid : GK_SID_OTHER;
    }
    default: return v.node != GK_NONE ? gk_x_sid_exotic(c, v) : (uint32_t)GK_SID_OTHER;
  }
}

GK_HD long long gk_x_numkey(const GkXCtx& c, const GkXVal& v) {
  if (v.vt == GK_VT_NUM) {
    if (v.node == GK_NONE) return 2 * v.inum;
    const gk_u64 e = c.doc.tape[v.node];
    return gk_num_key_token(c.doc.js + gk_te_off(e), gk_te_len(e));
  }
  // non-numbers: below (null, booleans) or above (strings, composites) every number -- OPA's cross-type order
  if (v.vt == GK_VT_NULL || v.vt == GK_VT_TRUE || v.vt == GK_VT_FALSE) return (long long)0x8000000000000000ull;
  return 0x7fffffffffffffffll;
}

// count() of a collection / string: elements, DISTINCT keys, code points
GK_HD bool gk_x_count(const GkXCtx& c, const GkXVal& v, long long* out) {
  if (v.vt == GK_VT_ARR && v.node != GK_NONE) {
    *out = gk_te_count(c.doc.tape[v.node]);
    return true;
  }
  if (v.vt == GK_VT_OBJ) {
    if (v.node == GK_NONE) {
      *out = 0;   // (synthetic envelope objects are not counted by any template; the host gives their true size)
      return false;
    }
    const uint32_t end = gk_te_end(c.doc.tape[v.node]);
    long long n = 0;
    for (uint32_t i = v.node + 1u; i < end; i = gk_tape_skip(c.doc.tape, i + 1u))
      if (!gk_key_shadowed(c.doc, i, end)) ++n;
    *out = n;
    return true;
  }
  if (v.vt == GK_VT_STR) {
    GkStr s = gk_x_str(c, v);
    long long n = 0;
    for (int b; (b = gk_str_next(s)) >= 0;)
      if ((b & 0xC0) != 0x80) ++n;
    *out = n;
    return true;
  }
  return false;
}

// hash + location of one Lut argument
GK_HD gk_u64 gk_x_arg(const GkXCtx& c, const GkXVal& v, gk_u64 h, GkMissArg* ma) {
  ma->kind = GK_ARG_UNDEF;
  ma->len = 0;
  ma->off = 0;
  if (v.vt == GK_VT_UNDEF) return gk_hash_byte(h, 0xF0u);
  if (v.node != GK_NONE) {
    const gk_u64 e = c.doc.tape[v.node];
    const uint32_t t = gk_te_type(e);
    uint32_t a, b;   // raw byte span of the value
    if (t == GK_T_OBJ || t == GK_T_ARR) {   // the sub-tree's raw text (its GK_T_END entry holds the byte span)
      const gk_u64 x = c.doc.tape[gk_te_end(e)];
      h = gk_hash_byte(h, t);
      h = gk_hash_bytes(h, c.doc.js + gk_te_off(x), gk_te_len(x));
      ma->kind = GK_ARG_JSON;
      ma->off = c.blob_off + gk_te_off(x);
      ma->len = gk_te_len(x);
      return h;
    }
    const uint32_t q = (t == GK_T_STR || t == GK_T_KEY) ? 1u : 0u;
    a = gk_te_off(e) - q;
    b = gk_te_off(e) + gk_te_len(e) + q;
    h = gk_hash_byte(h, t == GK_T_KEY ? (uint32_t)GK_T_STR : t);
    h = gk_hash_bytes(h, c.doc.js + gk_te_off(e), gk_te_len(e));
    ma->kind = GK_ARG_JSON;
    ma->off = c.blob_off + a;
    ma->len = b - a;
    return h;
  }
  if (v.vt == GK_VT_NUM) {
    h = gk_hash_byte(h, 0xF3u);
    for (int i = 0; i < 8; ++i) h = gk_hash_byte(h, (uint32_t)((unsigned long long)v.inum >> (8 * i)) & 0xffu);
    ma->kind = GK_ARG_INDEX;
    ma->off = (unsigned long long)v.inum;
    return h;
  }
  if (v.vt == GK_VT_STR) {
    h = gk_hash_byte(h, 0xF4u);
    h = gk_hash_bytes(h, v.sp, v.slen);
    ma->kind = GK_ARG_SYNSTR;
    ma->off = v.sp ? (unsigned long long)(c.blob_off + (unsigned long long)(v.sp - c.doc.js)) : 0ull;
    ma->len = v.slen;
    return h;
  }
  // other synthetic values (envelope objects / null) never reach a Lut (not leaf-like)
  h = gk_hash_byte(h, 0xF5u + v.vt);
  return h;
}

GK_HD uint32_t gk_x_sid_exotic(const GkXCtx& c, const GkXVal& v) {
  const uint32_t t = gk_te_type(c.doc.tape[v.node]);
  if (t == GK_T_OBJ || t == GK_T_ARR) {
    // a composite larger than 1 KiB never equals a parameter in practice: answered "other" without a lookup (documented limit)
    if (gk_te_len(c.doc.tape[gk_te_end(c.doc.tape[v.node])]) > 1024u) return GK_SID_OTHER;
  }
  GkMissArg ma;
  const gk_u64 h = gk_x_arg(c, v, GK_SEED_SIDVAL, &ma);
  const uint32_t ix = gk_lut_lookup(*c.xp, *static_cast<const GkIngestIn*>(c.in), GK_CL_SIDVAL, gk_hash_fin(h), &ma, 1);
  return ix == GK_HT_PENDING ? (uint32_t)GK_SID_OTHER : c.xp->lut_vals[ix].sid;
}

// ---------------------------------------------------------------------------------------------- native string closures
struct GkSV {
  uint32_t kind;          // 0 undefined, 1 string slice, 2 list = split(slice, delim), 3 number
  const uint8_t* p;
  uint32_t len;
  const uint8_t* d;
  uint32_t dlen;
  long long num;
};
GK_HD bool gk_sv_in_cutset(const uint8_t* cs, uint32_t n, uint32_t b) {
  for (uint32_t i = 0; i < n; ++i)
    if (cs[i] == b) return true;
  return false;
}
GK_HD uint32_t gk_sv_find(const uint8_t* p, uint32_t len, const uint8_t* d, uint32_t dlen, uint32_t from) {   // next occurrence or len
  for (uint32_t i = from; i + dlen <= len; ++i)
    if (p[i] == d[0] && gk_bytes_eq(p + i, d, dlen)) return i;
  return len;
}
// runs the program; false = not computable natively for this row (escaped leaf, non-ASCII cutset ...): use the lookup table
GK_HD bool gk_sx_run(const GkXCtx& c, const GkXClosure& cl, GkSV* out) {
  const GkXProg& xp = *c.xp;
  GkSV st[4];
  int sp = 0;
  for (uint32_t i = 0; i < cl.sx_n; ++i) {
    const uint32_t* op = xp.xkeys + cl.sx_off + 3u * i;
    switch (op[0]) {
      case GK_SX_LEAF: {
        if (sp >= 4) return false;
        const GkXVal v = gk_x_eval(c, xp.xargs[cl.args_off + op[1]]);
        GkSV& x = st[sp++];
        x.kind = 0;
        x.p = x.d = nullptr;
        x.len = x.dlen = 0;
        x.num = 0;
        if (v.vt == GK_VT_UNDEF) break;
        if (v.vt != GK_VT_STR) return false;              // (a non-string operand: the host words the type error / undefined)
        if (v.node != GK_NONE) {
          const gk_u64 e = c.doc.tape[v.node];
          if (gk_te_esc(e)) return false;
          x.p = c.doc.js + gk_te_off(e);
          x.len = gk_te_len(e);
        } else {
          if (v.sesc) return false;
          x.p = v.sp;
          x.len = v.slen;
        }
        for (uint32_t k = 0; k < x.len; ++k)
          if (x.p[k] >= 0x80u) return false;              // non-ASCII: rune semantics (trim cutsets, split("")) stay with the host
        x.kind = 1;
        break;
      }
      case GK_SX_SPLIT: {
        GkSV& x = st[sp - 1];
        if (x.kind == 0) break;
        if (x.kind != 1 || op[2] == 0) return false;
        x.kind = 2;
        x.d = xp.xbytes + op[1];
        x.dlen = op[2];
        break;
      }
      case GK_SX_TRIM: {
        GkSV& x = st[sp - 1];
        if (x.kind == 0) break;
        if (x.kind != 1) return false;
        const uint8_t* cs = xp.xbytes + op[1];
        while (x.len && gk_sv_in_cutset(cs, op[2], x.p[0])) ++x.p, --x.len;
        while (x.len && gk_sv_in_cutset(cs, op[2], x.p[x.len - 1])) --x.len;
        break;
      }
      case GK_SX_INDEX:
      case GK_SX_LAST: {
        GkSV& x = st[sp - 1];
        if (x.kind == 0) break;
        if (x.kind != 2) return false;
        uint32_t a = 0, seg = 0;
        bool found = false;
        for (;;) {
          const uint32_t b = gk_sv_find(x.p, x.len, x.d, x.dlen, a);
          const bool last = b == x.len;
          if (op[0] == GK_SX_LAST ? last : seg == op[1]) {
            x.p += a;
            x.len = b - a;
            found = true;
            break;
          }
          if (last) break;
          a = b + x.dlen;
          ++seg;
        }
        x.kind = found ? 1u : 0u;
        break;
      }
      case GK_SX_COUNT: {
        GkSV& x = st[sp - 1];
        if (x.kind == 0) break;
        if (x.kind == 1) {
          x.num = x.len;   // ASCII: bytes == code points
        } else if (x.kind == 2) {
          long long nseg = 1;
          for (uint32_t a = 0;;) {
            const uint32_t b = gk_sv_find(x.p, x.len, x.d, x.dlen, a);
            if (b == x.len) break;
            ++nseg;
            a = b + x.dlen;
          }
          x.num = nseg;
        } else {
          return false;
        }
        x.kind = 3;
        break;
      }
      default: return false;
    }
  }
  if (sp != 1) return false;
  *out = st[0];
  return true;
}

// ---------------------------------------------------------------------------------------------- one object
GK_HD uint32_t gk_decoded_len(const GkXCtx& c, const GkXVal& v) {
  if (v.node == GK_NONE) {
    if (!v.sesc) return v.slen;
  } else {
    const gk_u64 e = c.doc.tape[v.node];
    if (!gk_te_esc(e)) return gk_te_len(e);
  }
  GkStr s = gk_x_str(c, v);
  uint32_t n = 0;
  while (gk_str_next(s) >= 0) ++n;
  return n;
}
GK_HD void gk_copy_decoded(const GkXCtx& c, const GkXVal& v, uint8_t* dst) {
  GkStr s = gk_x_str(c, v);
  for (int b; (b = gk_str_next(s)) >= 0;) *dst++ = (uint8_t)b;
}
GK_HD bool gk_wild_val(const GkXCtx& c, uint32_t mode, const uint8_t* pat, uint32_t pl, const GkXVal& v) {
  // Wildcard.Matches (pkg/wildcard/wildcard.go:17-29) on a decoded name.  Names are DNS labels (<= 253 bytes); a longer one is
  // cut at 256 bytes, which only a prefix pattern can still match exactly.
  uint8_t buf[256];
  uint32_t n = 0;
  GkStr s = gk_x_str(c, v);
  int b;
  while (n < 256u && (b = gk_str_next(s)) >= 0) buf[n++] = (uint8_t)b;
  const bool cut = n == 256u && gk_str_next(s) >= 0;
  if (cut && mode != GK_W_PREFIX) return false;
  switch (mode) {
    case GK_W_PREFIX: return gk_prefix(buf, n, pat, pl);
    case GK_W_SUFFIX: return gk_suffix(buf, n, pat, pl);
    case GK_W_CONTAINS: return gk_contains(buf, n, pat, pl);
    default: return n == pl && gk_bytes_eq(buf, pat, pl);
  }
}

// the per-object working counters: contiguous on the host, strided by the object count on the device (coalesced)
struct GkCur {
  uint32_t* p;
  size_t stride;
  GK_HD uint32_t& operator[](uint32_t k) const { return p[(size_t)k * stride]; }
};

GK_HD const uint8_t* gk_lit(const char* s) { return reinterpret_cast<const uint8_t*>(s); }

// gk_emit_col<BCOLS>: the byte-encoded columns of a row (offsets = scanned lengths); <COLS>: every other column.
// gk_ingest_obj<COUNT / HEADER>: the two header passes.
enum { GK_PASS_COUNT = 0, GK_PASS_BCOLS = 1, GK_PASS_COLS = 2, GK_PASS_HEADER = 3 };
template <int MODE>
GK_HD void gk_emit_col(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, GkXCtx& c, uint32_t ci, uint32_t row, const GkCur& bcur) {
  const GkXCol& col = xp.cols[ci];
  const GkXClosure& cl = xp.cl[col.closure];
  const uint32_t enc = col.enc;
  if (MODE == GK_PASS_BCOLS && !(enc & GK_ENC_BYTES)) return;
  if (MODE == GK_PASS_COLS && (enc & GK_ENC_BYTES)) return;
  GkXVal v = gk_xundef();
  bool native = false;
  if (cl.kind == GK_X_LUT && cl.sx_n) {
    GkSV sv;
    if (gk_sx_run(c, cl, &sv)) {
      native = true;
      if (sv.kind == 1) v = gk_xstr(sv.p, sv.len);
      else if (sv.kind == 2) v = gk_xsyn(GK_VT_ARR);
      else if (sv.kind == 3) {
        v = gk_xsyn(GK_VT_NUM);
        v.inum = sv.num;
      }
    }
  }
  if (cl.kind == GK_X_LUT && !native) {
    GkMissArg ma[GK_LUT_MAX_ARGS];
    gk_u64 h = cl.seed;
    for (uint32_t a = 0; a < cl.nargs; ++a) h = gk_x_arg(c, gk_x_eval(c, xp.xargs[cl.args_off + a]), gk_hash_byte(h, 0xEEu), &ma[a]);
    const uint32_t ix = gk_lut_lookup(xp, in, col.closure, gk_hash_fin(h), ma, cl.nargs);
    GkLutVal lv;
    lv.vt = GK_VT_UNDEF;
    lv.sid = GK_SID_UNDEF;
    lv.num = 0;
    for (int w = 0; w < GK_HEAD_WORDS; ++w) lv.head[w] = 0;
    if (ix != GK_HT_PENDING) lv = xp.lut_vals[ix];
    if (enc & GK_ENC_VT) out.vt[ci][row] = (uint8_t)lv.vt;
    if (enc & GK_ENC_SID) out.sid[ci][row] = lv.sid;
    if (enc & GK_ENC_NUM) out.num[ci][row] = lv.num;
    if (enc & GK_ENC_HEAD)
      for (int w = 0; w < GK_HEAD_WORDS; ++w) out.head[ci][(size_t)row * GK_HEAD_WORDS + w] = lv.head[w];
    return;
  }
  if (native) {
    // (v holds the result)
  } else if (cl.kind == GK_X_COUNT) {
    const GkXVal b = gk_x_eval(c, (uint32_t)cl.base);
    long long n;
    if (gk_x_count(c, b, &n)) {
      v = gk_xsyn(GK_VT_NUM);
      v.inum = n;
    }
  } else {
    v = gk_x_eval(c, col.closure);
  }
  if (enc & GK_ENC_VT) out.vt[ci][row] = (uint8_t)v.vt;
  if (enc & GK_ENC_SID) out.sid[ci][row] = gk_x_sid(c, v);
  if (enc & GK_ENC_NUM) out.num[ci][row] = v.vt == GK_VT_UNDEF ? 0ll : gk_x_numkey(c, v);
  if (enc & GK_ENC_HEAD) {
    uint32_t h[GK_HEAD_WORDS];
    for (int w = 0; w < GK_HEAD_WORDS; ++w) h[w] = 0;
    if (v.vt == GK_VT_STR) {
      GkStr s = gk_x_str(c, v);
      uint32_t n = 0;
      for (int b; (b = gk_str_next(s)) >= 0; ++n)
        if (n < GK_HEAD_BYTES) h[n >> 2] |= (uint32_t)b << (8u * (n & 3u));
      h[GK_HEAD_WORDS - 1] |= (n < 255u ? n : 255u) << 24;
    }
    for (int w = 0; w < GK_HEAD_WORDS; ++w) out.head[ci][(size_t)row * GK_HEAD_WORDS + w] = h[w];
  }
  if (enc & GK_ENC_BYTES) {   // (the offsets are there already: the scanned lengths of gk_bcol_len)
    (void)bcur;
    if (v.vt == GK_VT_STR) gk_copy_decoded(c, v, out.bytes[ci] + out.boff[ci][row]);
  }
}

// The header pass of one object.  COUNT fills in.counts[k * n + i] (k: name bytes, generateName bytes, labels, nsname bytes);
// HEADER finds the exclusive prefix sums there.  `cur`: GK_CNT_EXTRA working counters private to the thread.
template <int MODE>
GK_HD void gk_ingest_obj(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t i, const GkCur& cur, uint32_t lane, uint32_t nlanes) {
  // The header of object i -- every thread runs the same steps in the same order.  COUNT: byte / label counts of the header
  // arrays (+ the flags word into out.flags, a scratch array at that point).  HEADER: the header arrays themselves, at the
  // scanned offsets.  Scopes and columns are level-synchronous passes of their own (gk_scope_count ... gk_bcol_write).
  constexpr bool WRITE = MODE != GK_PASS_COUNT;
  constexpr bool HDR = true;
  const uint32_t n = in.n, NK = GK_CNT_EXTRA;
  const uint32_t K_NAME = 0, K_GEN = 1, K_LBL = 2, K_NSN = 3;
  for (uint32_t k = 0; k < NK; ++k) cur[k] = WRITE ? in.counts[(size_t)k * n + i] : 0u;
  GkXCtx c;
  c.xp = &xp;
  c.in = &in;
  c.blob_off = in.ooff[i];
  c.doc.js = in.blob + in.ooff[i];
  c.doc.tape = in.tape + gk_tape_off(in.ooff, i);
  c.doc.ntape = in.ntape[i];
  c.depth = 0;
  c.scope_at[0] = 0;
  c.env_ready = 0;
  c.memo = nullptr;
  c.api_node = c.kind_node = c.name_node = c.ns_node = c.meta_node = GK_NONE;
  c.grp = c.ver = nullptr;
  c.grp_len = c.ver_len = 0;
  bool skip = in.status[i] != GK_ING_OK;
  uint32_t fl = (in.source << GK_F_SRC_SHIFT) & GK_F_SRC_MASK;
  uint32_t kind_sid = GK_SID_UNDEF, group_sid = GK_SID_UNDEF, nsrow = GK_NONE;
  uint32_t labels = GK_NONE, gen_node = GK_NONE;
  GkXVal nsname = gk_xundef();
  if (HDR && !skip) {
    // ---- review envelope / header: apiVersion -> (group, version), kind, metadata.{name, generateName, namespace, labels}
    gk_x_envelope(c);
    const uint32_t meta = c.meta_node, nm = c.name_node, ns = c.ns_node;
    if (meta != GK_NONE) {
      gen_node = gk_obj_find(c.doc, meta, gk_lit("generateName"), 12);
      labels = gk_obj_find(c.doc, meta, gk_lit("labels"), 6);
      if (gen_node != GK_NONE && (gk_te_type(c.doc.tape[gen_node]) != GK_T_STR || gk_te_len(c.doc.tape[gen_node]) == 0)) gen_node = GK_NONE;
      if (labels != GK_NONE && gk_te_type(c.doc.tape[labels]) != GK_T_OBJ) labels = GK_NONE;
    }
    const GkXVal kindv = gk_xnode(c.doc.tape, c.kind_node);
    const bool is_ns = c.grp_len == 0 && gk_entry_eq(c.doc, c.doc.tape[c.kind_node], gk_lit("Namespace"), 9);
    // ---- stage 0: the process excluder (pkg/controller/config/process/excluder.go:95-127): a Namespace by its own name,
    // anything else by its namespace ("" for cluster-scoped objects)
    if (xp.excl_n) {
      const GkXVal subject = is_ns ? (nm != GK_NONE ? gk_xnode(c.doc.tape, nm) : gk_xstr(nullptr, 0)) : (ns != GK_NONE ? gk_xnode(c.doc.tape, ns) : gk_xstr(nullptr, 0));
      for (uint32_t j = 0; j < xp.excl_n && !skip; ++j) {
        const uint32_t* e = xp.xkeys + xp.excl_off + 3u * j;
        skip = gk_wild_val(c, e[0], xp.xbytes + e[1], e[2], subject);
      }
    }
    if (!skip) {
      fl |= GK_F_HAS_OBJ;
      if (is_ns) fl |= GK_F_IS_NS;
      if (ns != GK_NONE) fl |= GK_F_HAS_NS;
      if (MODE == GK_PASS_HEADER) {
        kind_sid = gk_x_sid(c, kindv);
        group_sid = gk_x_sid(c, gk_xstr_esc(c.grp, c.grp_len, c.env_esc));
      }
      if (ns != GK_NONE) {   // the Namespace object of the review: the cache entry for the object's namespace (matcher.go:37-39)
        GkStr s = gk_x_str(c, gk_xnode(c.doc.tape, ns));
        gk_u64 h = GK_SEED_NS;
        for (int b; (b = gk_str_next(s)) >= 0;) h = gk_hash_byte(h, (uint32_t)b);
        bool present;
        const uint32_t r = gk_ht_find(xp.ns_tab, gk_hash_fin(h), &present);
        if (present) {
          nsrow = r;
          fl |= GK_F_NS_OBJ;
        }
      }
      // the name namespaces / excludedNamespaces match on (match.go:118-179)
      if (is_ns) nsname = nm != GK_NONE ? gk_xnode(c.doc.tape, nm) : gk_xstr(nullptr, 0);
      else if (nsrow != GK_NONE) nsname = gk_xstr(xp.nsn_bytes + xp.nsn_off[nsrow], xp.nsn_off[nsrow + 1] - xp.nsn_off[nsrow]);
      else if (ns != GK_NONE) nsname = gk_xnode(c.doc.tape, ns);
      if (nsname.vt != GK_VT_UNDEF) fl |= GK_F_NSNAME;
    }
  }
  if (skip) fl = (fl & GK_F_SRC_MASK) | GK_F_SKIP;
  // ---- header arrays
  if (HDR) {
    const GkXVal namev = (!skip && c.name_node != GK_NONE) ? gk_xnode(c.doc.tape, c.name_node) : gk_xundef();
    const GkXVal genv = (!skip && gen_node != GK_NONE) ? gk_xnode(c.doc.tape, gen_node) : gk_xundef();
    if (MODE == GK_PASS_HEADER && lane == 0) {
      if (out.gvk) {
        gk_u64 hh = 0;
        if (!skip) {
          // of the decoded strings, so that spellings of one (apiVersion, kind) share the hash
          hh = 0x9ae16a3b2f90404full;
          if (c.api_node != GK_NONE && gk_te_type(c.doc.tape[c.api_node]) == GK_T_STR) hh = gk_hash_entry(c.doc, c.doc.tape[c.api_node], hh);
          hh = gk_hash_byte(hh, 0xFFu);
          hh = gk_hash_fin(gk_hash_entry(c.doc, c.doc.tape[c.kind_node], hh)) | 1ull;
        }
        out.gvk[i] = hh;
      }
      out.flags[i] = fl;
      out.kind_sid[i] = kind_sid;
      out.group_sid[i] = group_sid;
      out.nsrow[i] = nsrow;
      out.name_off[i] = cur[K_NAME];
      out.gen_off[i] = cur[K_GEN];
      out.lbl_off[i] = cur[K_LBL];
      out.nsn_off[i] = cur[K_NSN];
      if (namev.vt == GK_VT_STR) gk_copy_decoded(c, namev, out.name_bytes + cur[K_NAME]);
      if (genv.vt == GK_VT_STR) gk_copy_decoded(c, genv, out.gen_bytes + cur[K_GEN]);
      if (nsname.vt == GK_VT_STR) gk_copy_decoded(c, nsname, out.nsn_bytes + cur[K_NSN]);
    }
    if (namev.vt == GK_VT_STR) cur[K_NAME] += gk_decoded_len(c, namev);
    if (genv.vt == GK_VT_STR) cur[K_GEN] += gk_decoded_len(c, genv);
    if (nsname.vt == GK_VT_STR) cur[K_NSN] += gk_decoded_len(c, nsname);
    if (!skip && labels != GK_NONE) {
      const uint32_t end = gk_te_end(c.doc.tape[labels]);
      for (uint32_t k = labels + 1u; k < end; k = gk_tape_skip(c.doc.tape, k + 1u)) {
        if (gk_key_shadowed(c.doc, k, end)) continue;
        if (MODE == GK_PASS_HEADER && lane == 0) {
          const GkXVal val = gk_xnode(c.doc.tape, k + 1u);
          out.lbl_kv[2u * (size_t)cur[K_LBL]] = gk_x_sid(c, gk_xnode(c.doc.tape, k));
          out.lbl_kv[2u * (size_t)cur[K_LBL] + 1u] = val.vt == GK_VT_STR ? gk_x_sid(c, val) : GK_SID_OTHER;
        }
        ++cur[K_LBL];
      }
    }
    if (MODE == GK_PASS_HEADER && lane == 0 && i + 1u == n) {
      out.name_off[n] = cur[K_NAME];
      out.gen_off[n] = cur[K_GEN];
      out.lbl_off[n] = cur[K_LBL];
      out.nsn_off[n] = cur[K_NSN];
    }
  }
  if (MODE == GK_PASS_COUNT && lane == 0) {
    // header counters (scanned next) + the flags word: the scope passes read the skip bit before the arena exists
    for (uint32_t k = 0; k < NK; ++k) in.counts[(size_t)k * n + i] = cur[k];
    out.flags[i] = fl;
  }
}


// ---------------------------------------------------------------------------------------------- level-synchronous passes
// Scopes are filled level by level: for scope t, one thread per row of its PARENT scope counts the members of the generator
// collection (gk_scope_count), a device scan of the counts is the CSR offset array, and a second pass writes one 16-byte row
// handle per member (gk_scope_fill).  Threads of a warp then always work on the same scope, the same generator path and the
// same columns -- unlike a per-object walk of the whole scope tree, where every thread is somewhere else.

// evaluation context of row r of scope sc (scope 0: r is the object); returns the object index
GK_HD uint32_t gk_row_ctx(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t sc, uint32_t r, GkXCtx& c) {
  GkRowRec me;
  me.elem = me.key = me.parent = 0;
  me.obj = r;
  if (sc) me = out.row_rec[sc][r];
  const uint32_t i = me.obj;
  c.xp = &xp;
  c.in = &in;
  c.blob_off = in.ooff[i];
  c.doc.js = in.blob + in.ooff[i];
  c.doc.tape = in.tape + gk_tape_off(in.ooff, i);
  c.doc.ntape = in.ntape[i];
  c.env_ready = 0;
  c.memo = nullptr;
  c.api_node = c.kind_node = c.name_node = c.ns_node = c.meta_node = GK_NONE;
  c.grp = c.ver = nullptr;
  c.grp_len = c.ver_len = 0;
  c.scope_at[0] = 0;
  int d = 0;
  for (uint32_t s2 = sc; s2; s2 = (uint32_t)xp.scopes[s2].parent) ++d;
  c.depth = d;
  uint32_t cs = sc;
  GkRowRec rr = me;
  for (int dd = d; dd >= 1; --dd) {
    c.scope_at[dd] = cs;
    c.elem_node[dd] = rr.elem;
    c.key_ref[dd] = rr.key;
    cs = (uint32_t)xp.scopes[cs].parent;
    if (cs) rr = out.row_rec[cs][rr.parent];
  }
  return i;
}

// rows of scope t under row r of its parent scope; *coll = tape index of the generator collection (GK_NONE: no rows)
GK_HD uint32_t gk_scope_count(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t t, uint32_t r, uint32_t* coll_out) {
  *coll_out = GK_NONE;
  const uint32_t p = (uint32_t)xp.scopes[t].parent;
  GkXCtx c;
  const uint32_t i = gk_row_ctx(xp, in, out, p, r, c);
  if ((out.flags[i] & GK_F_SKIP) || c.depth >= GK_MAX_LOOP_DEPTH) return 0u;
  const GkXVal coll = gk_x_eval(c, xp.scopes[t].gen);
  if (coll.node == GK_NONE || (coll.vt != GK_VT_ARR && coll.vt != GK_VT_OBJ)) return 0u;
  *coll_out = coll.node;
  const gk_u64 e = c.doc.tape[coll.node];
  if (coll.vt == GK_VT_ARR) return gk_te_count(e);
  // object members: a key repeated later in the same object is shadowed by the later one
  const uint32_t end = gk_te_end(e);
  uint32_t cnt = 0;
  for (uint32_t k = coll.node + 1u; k < end; k = gk_tape_skip(c.doc.tape, k + 1u))
    if (!gk_key_shadowed(c.doc, k, end)) ++cnt;
  return cnt;
}

// the row handles of scope t under parent row r, from row `first` on (rows of a scope are in (parent row, member) order)
GK_HD void gk_scope_fill(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t t, uint32_t r, uint32_t coll, uint32_t first) {
  if (coll == GK_NONE) return;
  const uint32_t p = (uint32_t)xp.scopes[t].parent;
  uint32_t i = r;
  if (p) i = out.row_rec[p][r].obj;
  const gk_u64* tape = in.tape + gk_tape_off(in.ooff, i);
  const gk_u64 e = tape[coll];
  const uint32_t end = gk_te_end(e);
  GkRowRec rr;
  rr.parent = r;
  rr.obj = i;
  uint32_t row = first;
  if (gk_te_type(e) == GK_T_ARR) {
    uint32_t ix = 0;
    for (uint32_t k = coll + 1u; k < end; k = gk_tape_skip(tape, k)) {
      rr.elem = k;
      rr.key = ix++ | GK_ROW_INDEX;
#ifdef __CUDA_ARCH__
      *reinterpret_cast<uint4*>(&out.row_rec[t][row]) = *reinterpret_cast<const uint4*>(&rr);
#else
      out.row_rec[t][row] = rr;
#endif
      ++row;
    }
  } else {
    GkDoc d;
    d.js = in.blob + in.ooff[i];
    d.tape = tape;
    d.ntape = in.ntape[i];
    for (uint32_t k = coll + 1u; k < end; k = gk_tape_skip(tape, k + 1u)) {
      if (gk_key_shadowed(d, k, end)) continue;
      rr.elem = k + 1u;
      rr.key = k;
#ifdef __CUDA_ARCH__
      *reinterpret_cast<uint4*>(&out.row_rec[t][row]) = *reinterpret_cast<const uint4*>(&rr);
#else
      out.row_rec[t][row] = rr;
#endif
      ++row;
    }
  }
}

// decoded byte length of byte-encoded column ci at row r of its scope
GK_HD uint32_t gk_bcol_len(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t ci, uint32_t r) {
  const GkXCol& col = xp.cols[ci];
  const GkXClosure& cl = xp.cl[col.closure];
  if (cl.kind == GK_X_LUT || cl.kind == GK_X_COUNT) return 0u;   // (never strings with bytes: values of a lookup / a count)
  GkXCtx c;
  const uint32_t i = gk_row_ctx(xp, in, out, (uint32_t)col.scope, r, c);
  if (out.flags[i] & GK_F_SKIP) return 0u;
  const GkXVal v = gk_x_eval(c, col.closure);
  return v.vt == GK_VT_STR ? gk_decoded_len(c, v) : 0u;
}

// every encoding of byte-encoded column ci at row r (the offsets array is in place: scanned lengths)
GK_HD void gk_bcol_write(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t ci, uint32_t r) {
  const GkXCol& col = xp.cols[ci];
  GkXCtx c;
  const uint32_t i = gk_row_ctx(xp, in, out, (uint32_t)col.scope, r, c);
  if (out.flags[i] & GK_F_SKIP) {   // placeholder row (scope 0 only: a skipped object has no other rows)
    const uint32_t enc = col.enc;
    if (enc & GK_ENC_VT) out.vt[ci][r] = GK_VT_UNDEF;
    if (enc & GK_ENC_SID) out.sid[ci][r] = GK_SID_UNDEF;
    if (enc & GK_ENC_NUM) out.num[ci][r] = 0;
    if (enc & GK_ENC_HEAD)
      for (int w = 0; w < GK_HEAD_WORDS; ++w) out.head[ci][(size_t)r * GK_HEAD_WORDS + w] = 0;
    return;
  }
  const GkCur none{nullptr, 0};
  gk_emit_col<GK_PASS_BCOLS>(xp, in, out, c, ci, r, none);
}

// The per-row column pass: every column of scope `sc` that is not byte-encoded, for row `r` (scope 0: r = the object).
GK_HD void gk_ingest_row(const GkXProg& xp, const GkIngestIn& in, const GkIngestOut& out, uint32_t sc, uint32_t r, uint32_t lane, uint32_t nlanes) {
  GkXCtx c;
  const uint32_t i = gk_row_ctx(xp, in, out, sc, r, c);
  const GkXScope& xs = xp.scopes[sc];
  if (sc == 0 && (out.flags[i] & GK_F_SKIP)) {   // placeholder row: every encoding "undefined"
    for (uint32_t k = lane; k < xs.ncols; k += nlanes) {
      const uint32_t ci = xp.col_order[xs.first_col + k];
      const uint32_t enc = xp.cols[ci].enc;
      if (enc & GK_ENC_BYTES) continue;
      if (enc & GK_ENC_VT) out.vt[ci][i] = GK_VT_UNDEF;
      if (enc & GK_ENC_SID) out.sid[ci][i] = GK_SID_UNDEF;
      if (enc & GK_ENC_NUM) out.num[ci][i] = 0;
      if (enc & GK_ENC_HEAD)
        for (int w = 0; w < GK_HEAD_WORDS; ++w) out.head[ci][(size_t)i * GK_HEAD_WORDS + w] = 0;
    }
    return;
  }
  // the columns of a row share path prefixes (`resources`, `resources.limits`, `resources.limits.cpu` ...): each step once
  unsigned short memo[GK_MEMO_MAX];
  if (xp.ncl <= GK_MEMO_MAX) {
    for (uint32_t k = 0; k < xp.ncl; ++k) memo[k] = GK_MEMO_EMPTY;
    c.memo = memo;
  }
  const GkCur none{nullptr, 0};
  for (uint32_t k = lane; k < xs.ncols; k += nlanes) gk_emit_col<GK_PASS_COLS>(xp, in, out, c, xp.col_order[xs.first_col + k], r, none);
}

// tokenise object i of the chunk and run the review-level checks of Engine::review_doc (the object must be a JSON object
// with a non-empty string `kind`; a literal null is "no object")
GK_HD void gk_tape_obj(const GkIngestIn& in, uint32_t i) {
  const unsigned long long a = in.ooff[i], b = in.ooff[i + 1];
  unsigned long long* tape = in.tape + gk_tape_off(in.ooff, i);
  uint32_t nt = 0;
  int st = (b - a > 0xfffffff0ull) ? (int)GK_ING_TOO_LONG : gk_tape_build(in.blob + a, (uint32_t)(b - a), tape, gk_tape_capacity(b - a), &nt);
  if (st == GK_ING_OK) {
    const uint32_t t0 = gk_te_type(tape[0]);
    if (t0 == GK_T_NULL) st = GK_ING_NULL;
    else if (t0 != GK_T_OBJ) st = GK_ING_NOT_OBJECT;
    else {
      GkDoc d;
      d.js = in.blob + a;
      d.tape = tape;
      d.ntape = nt;
      const uint32_t k = gk_obj_find(d, 0, reinterpret_cast<const uint8_t*>("kind"), 4);
      if (k == GK_NONE || gk_te_type(tape[k]) != GK_T_STR || gk_te_len(tape[k]) == 0) st = GK_ING_NO_KIND;
    }
  }
  in.ntape[i] = nt;
  in.status[i] = (uint32_t)st;
}
