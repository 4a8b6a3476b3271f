// Host side of the device ingest path (ingest_core.h): the extraction program built from a compiled Schema, the lookup
// tables (string -> sid, namespace cache, Lut results) in their host form, and the request a backend's ingest() takes.
#pragma once
#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "ingest_core.h"
#include "lower.hpp"

namespace gk {

class StringTable;
struct Compiled;

struct XProgHost {
  std::vector<GkXClosure> cl;
  std::vector<CP> cl_src;                          // the schema closure behind each entry (null: an internal argument path)
  std::vector<std::vector<XInfo::Arg>> cl_args;    // Lut entries: the normalised leaf arguments, in xargs order
  std::vector<GkXCol> cols;
  std::vector<GkXScope> scopes;
  std::vector<uint32_t> col_order, xkeys, xargs;
  std::vector<uint8_t> xbytes;
  uint32_t nbytecols = 0;
  uint32_t ncounters() const { return (uint32_t)scopes.size() + nbytecols + GK_CNT_EXTRA; }
};
// throws RegoError when a scope / column cannot be computed by the ingest kernels
std::shared_ptr<const XProgHost> build_xprog(const Schema& s);

struct HashTabHost {
  std::vector<unsigned long long> keys;
  std::vector<uint32_t> vals;
  uint32_t mask = 0, used = 0;
  void init(uint32_t capacity_pow2) {
    keys.assign(capacity_pow2, 0ull);
    vals.assign(capacity_pow2, GK_HT_PENDING);
    mask = capacity_pow2 - 1;
    used = 0;
  }
  // returns the slot; an existing key keeps its slot (value overwritten)
  uint32_t put(unsigned long long key, uint32_t val) {
    uint32_t i = (uint32_t)key & mask;
    while (keys[i] != 0ull && keys[i] != key) i = (i + 1u) & mask;
    if (keys[i] == 0ull) ++used;
    keys[i] = key;
    vals[i] = val;
    return i;
  }
  GkHtab view() {
    GkHtab t;
    t.keys = keys.data();
    t.vals = vals.data();
    t.mask = mask;
    t.pad_ = 0;
    return t;
  }
};

// interned constants as a hash table: decoded string bytes / canonical integer text -> sid
struct SidTable {
  HashTabHost tab;
  uint32_t sid_true = GK_SID_OTHER, sid_false = GK_SID_OTHER, sid_null = GK_SID_OTHER;
  uint32_t nstrings = 0;   // size of the string table it was built from
};
void build_sid_table(const StringTable& st, SidTable& out);

// the namespace cache (pkg/target/ns_cache.go) as device tables: name -> row, labels per row, metadata.name per row
struct NsTableHost {
  HashTabHost tab;
  std::vector<uint32_t> nsl_off{0}, nsl_kv, nsn_off{0};
  std::vector<uint8_t> nsn_bytes;
};

struct IngestReq {
  const uint8_t* blob = nullptr;
  const unsigned long long* ooff = nullptr;   // [n + 1]
  size_t n = 0;
  uint32_t source = 0;                        // GK_SRC_*
  const Compiled* c = nullptr;
  std::shared_ptr<const XProgHost> xprog;
  const StringTable* strings = nullptr;
  std::shared_ptr<const NsTableHost> ns;
  std::vector<std::string> excluded;          // excluder patterns of the calling process
  // host evaluation of the lookups the device missed: one GkLutVal per record, in order; the records' argument spans are byte
  // offsets into `blob`
  std::function<void(const GkMiss* misses, size_t n, std::vector<GkLutVal>& out)> lut_fill;
  // the same with the spans read from `bytes` instead: a refresh from a kept source has no caller's page (Backend::reextract)
  std::function<void(const uint8_t* bytes, const GkMiss* misses, size_t n, std::vector<GkLutVal>& out)> lut_fill_from;
};

struct IngestStats {
  double h2d_ms = 0, tape_ms = 0, extract_ms = 0, lut_ms = 0, total_ms = 0;
  unsigned long long h2d_bytes = 0, lut_misses = 0, alg_bytes = 0, launches = 0;
};

// FNV + finaliser over host bytes (same function as the device's)
inline unsigned long long xhash(unsigned long long seed, const void* p, size_t n) {
  return gk_hash_fin(gk_hash_bytes(seed, static_cast<const uint8_t*>(p), (uint32_t)n));
}

}  // namespace gk
