// alloc_probe.c — LD_PRELOAD probe used by tools/monte_carlo_timing.py (measurement support, not part of the library).
// Interposes three calls of a process that runs the engine and appends one line per event to $OVB_ALLOC_LOG:
//   create <device bytes taken by ovb_create (cudaMemGetInfo before and after)>
//   malloc <ovb_msckf_update calls this thread has made> <bytes> <offset of the call site in its object> <object path>
// for every cudaMalloc made outside ovb_create, i.e. the buffers the engine grows on demand. The call-site offset is
// mapped to a function of libovb200.so with its symbol table (nm), which names the growth site.
// Build: cc -shared -fPIC -O2 -o alloc_probe.so alloc_probe.c -ldl
#define _GNU_SOURCE
#include <dlfcn.h>
#include <pthread.h>
#include <stdarg.h>
#include <stddef.h>
#include <stdio.h>
#include <stdlib.h>

typedef int cudaError_t;

static __thread int in_create;
static __thread long n_updates;
static pthread_mutex_t log_lock = PTHREAD_MUTEX_INITIALIZER;

static void *next_sym(const char *name) {
  void *p = dlsym(RTLD_NEXT, name);
  if (!p) {
    fprintf(stderr, "alloc_probe: %s not found\n", name);
    abort();
  }
  return p;
}

static void log_line(const char *fmt, ...) __attribute__((format(printf, 1, 2)));
static void log_line(const char *fmt, ...) {
  const char *path = getenv("OVB_ALLOC_LOG");
  if (!path)
    return;
  pthread_mutex_lock(&log_lock);
  FILE *f = fopen(path, "a");
  if (f) {
    va_list ap;
    va_start(ap, fmt);
    vfprintf(f, fmt, ap);
    va_end(ap);
    fclose(f);
  }
  pthread_mutex_unlock(&log_lock);
}

cudaError_t cudaMalloc(void **ptr, size_t bytes) {
  cudaError_t (*real)(void **, size_t) = (cudaError_t(*)(void **, size_t))next_sym("cudaMalloc");
  const cudaError_t e = real(ptr, bytes);
  if (!in_create) {
    Dl_info info;
    void *ra = __builtin_return_address(0);
    if (dladdr(ra, &info) && info.dli_fname)
      log_line("malloc %ld %zu %lu %s\n", n_updates, bytes, (unsigned long)((char *)ra - (char *)info.dli_fbase), info.dli_fname);
    else
      log_line("malloc %ld %zu 0 ?\n", n_updates, bytes);
  }
  return e;
}

int ovb_create(const void *cfg, void **out) {
  int (*real)(const void *, void **) = (int (*)(const void *, void **))next_sym("ovb_create");
  cudaError_t (*meminfo)(size_t *, size_t *) = (cudaError_t(*)(size_t *, size_t *))next_sym("cudaMemGetInfo");
  size_t free0 = 0, free1 = 0, total = 0;
  meminfo(&free0, &total);
  in_create = 1;
  const int st = real(cfg, out);
  in_create = 0;
  meminfo(&free1, &total);
  log_line("create %lld\n", (long long)free0 - (long long)free1);
  return st;
}

int ovb_msckf_update(void *ctx, const void *frame, const void *feats, const void *opts, void *out, double *dx, void *stats) {
  int (*real)(void *, const void *, const void *, const void *, void *, double *, void *) =
      (int (*)(void *, const void *, const void *, const void *, void *, double *, void *))next_sym("ovb_msckf_update");
  n_updates++;
  return real(ctx, frame, feats, opts, out, dx, stats);
}
