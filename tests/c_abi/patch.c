/* tests/c_abi/patch.c -- the Go shim's PatchBatch (go/gpudriver/audit.go) repeated call for call in C: the added documents copied
 * into one malloc'd page with its offsets, the drop indices into C memory, then gk_batch_patch.  Input lines (each payload followed by
 * a newline):
 *   T <kind> <len>\n<rego>   C <len>\n<constraint json>   D <len>\n<document of the page>   A <len>\n<added document>   X <index to drop>
 * Output: "N <size>" after the patch; "P <object> <words...>" the patched batch's violation plane and "F ..." a fresh upload's of the
 * resulting page; then the return codes of three refused calls and the size after them. */
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/gk_engine.h"

#define SYM(name) __typeof__(&name) p_##name = (__typeof__(&name))dlsym(lib, #name); if (!p_##name) { fprintf(stderr, "missing symbol %s\n", #name); return 2; }

typedef struct {
  char* buf;
  uint64_t* off;
  size_t n, bytes;
} page_t;

static void page_add(page_t* p, const char* doc, size_t len) {
  p->buf = (char*)realloc(p->buf, p->bytes + len + 1);
  p->off = (uint64_t*)realloc(p->off, (p->n + 2) * sizeof(uint64_t));
  if (p->n == 0) p->off[0] = 0;
  memcpy(p->buf + p->bytes, doc, len);
  p->bytes += len;
  p->off[++p->n] = p->bytes;
}

static char* read_n(FILE* f, size_t n) {
  char* b = (char*)malloc(n + 1);
  if (n && fread(b, 1, n, f) != n) { fprintf(stderr, "short read\n"); exit(2); }
  b[n] = 0;
  fgetc(f); /* newline */
  return b;
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  void* lib = dlopen(argv[1], RTLD_NOW | RTLD_LOCAL);
  if (!lib) { fprintf(stderr, "dlopen: %s\n", dlerror()); return 2; }
  SYM(gk_engine_create) SYM(gk_engine_destroy) SYM(gk_add_template) SYM(gk_add_constraint) SYM(gk_batch_upload_blob) SYM(gk_batch_patch)
  SYM(gk_batch_eval) SYM(gk_batch_size) SYM(gk_batch_free) SYM(gk_free_result) SYM(gk_free_str)
  FILE* f = fopen(argv[2], "rb");
  if (!f) return 2;
  char* err = NULL;
  gk_cfg cfg;
  memset(&cfg, 0, sizeof cfg);
  gk_engine_t* e = p_gk_engine_create(&cfg, &err);
  if (!e) { fprintf(stderr, "create: %s\n", err ? err : "?"); return 3; }
  page_t page = {0}, added = {0};
  uint32_t drop[256];
  size_t n_drop = 0;
  char tag;
  while (fscanf(f, " %c", &tag) == 1) {
    size_t len;
    if (tag == 'T') {
      char kind[256];
      if (fscanf(f, "%255s %zu", kind, &len) != 2) return 2;
      fgetc(f);
      char* rego = read_n(f, len);
      if (p_gk_add_template(e, kind, rego, len, &err)) { fprintf(stderr, "template: %s\n", err); return 3; }
      free(rego);
    } else if (tag == 'C' || tag == 'D' || tag == 'A') {
      if (fscanf(f, "%zu", &len) != 1) return 2;
      fgetc(f);
      char* js = read_n(f, len);
      if (tag == 'C' && p_gk_add_constraint(e, js, len, &err)) { fprintf(stderr, "constraint: %s\n", err); return 3; }
      if (tag != 'C') page_add(tag == 'D' ? &page : &added, js, len);
      free(js);
    } else if (tag == 'X') {
      unsigned x;
      if (fscanf(f, "%u", &x) != 1 || n_drop == 256) return 2;
      drop[n_drop++] = x;
    }
  }
  gk_batch_t* b = NULL;
  if (p_gk_batch_upload_blob(e, page.buf, page.off, page.n, GK_SOURCE_ORIGINAL, GK_F_KEEP_SOURCE, &b, NULL, &err)) { fprintf(stderr, "upload: %s\n", err); return 3; }
  /* PatchBatch: the documents in C memory that stays alive while the batch lives, the drop indices in C memory for the call */
  uint32_t* cdrop = (uint32_t*)malloc((n_drop + 1) * sizeof(uint32_t));
  memcpy(cdrop, drop, n_drop * sizeof(uint32_t));
  int rc = p_gk_batch_patch(e, b, cdrop, n_drop, added.buf, added.off, added.n, NULL, &err);
  free(cdrop);
  if (rc < 0) { fprintf(stderr, "patch: %s\n", err); return 3; }
  printf("N\t%d\n", rc);
  /* the resulting page, uploaded fresh */
  page_t result = {0};
  for (size_t i = 0; i < page.n; ++i) {
    int gone = 0;
    for (size_t k = 0; k < n_drop; ++k) gone |= drop[k] == i;
    if (!gone) page_add(&result, page.buf + page.off[i], (size_t)(page.off[i + 1] - page.off[i]));
  }
  for (size_t i = 0; i < added.n; ++i) page_add(&result, added.buf + added.off[i], (size_t)(added.off[i + 1] - added.off[i]));
  gk_batch_t* fresh = NULL;
  if (p_gk_batch_upload_blob(e, result.buf, result.off, result.n, GK_SOURCE_ORIGINAL, 0, &fresh, NULL, &err)) { fprintf(stderr, "fresh: %s\n", err); return 3; }
  gk_batch_t* which[2] = {b, fresh};
  for (int w = 0; w < 2; ++w) {
    gk_result res;
    if (p_gk_batch_eval(e, which[w], "audit.gatekeeper.sh", GK_F_BITMAP_ONLY, &res, &err)) { fprintf(stderr, "eval: %s\n", err); return 3; }
    for (uint32_t o = 0; o < res.n_objects; ++o) {
      printf("%c\t%u", w ? 'F' : 'P', o);
      for (uint32_t k = 0; k < res.words; ++k) printf("\t%u", res.viol_bits[(size_t)o * res.words + k]);
      printf("\n");
    }
    p_gk_free_result(&res);
  }
  /* refused calls: a duplicate index, an index out of range, a batch without a kept source */
  uint32_t dup[2] = {0, 0}, oor[1] = {(uint32_t)rc};
  err = NULL;
  printf("DUP\t%d\n", p_gk_batch_patch(e, b, dup, 2, NULL, NULL, 0, NULL, &err));
  p_gk_free_str(err);
  err = NULL;
  printf("RANGE\t%d\n", p_gk_batch_patch(e, b, oor, 1, NULL, NULL, 0, NULL, &err));
  p_gk_free_str(err);
  err = NULL;
  printf("NOSOURCE\t%d\n", p_gk_batch_patch(e, fresh, dup, 1, NULL, NULL, 0, NULL, &err));
  p_gk_free_str(err);
  printf("SIZE\t%u\n", p_gk_batch_size(b));
  p_gk_batch_free(e, b);
  p_gk_batch_free(e, fresh);
  p_gk_engine_destroy(e);
  return 0;
}
