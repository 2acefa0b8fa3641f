// common.cuh — context, scratch arena and error plumbing shared by the libb200feat kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/b2f.h"

namespace b2f {

void set_error(const char *fmt, ...);

#define B2F_CUDA(expr)                                                                     \
  do {                                                                                     \
    cudaError_t e__ = (expr);                                                              \
    if (e__ != cudaSuccess) {                                                              \
      b2f::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
      return B2F_ECUDA;                                                                    \
    }                                                                                      \
  } while (0)

#define B2F_LAUNCH_CHECK(ctx)                                                              \
  do {                                                                                     \
    (ctx)->launches++;                                                                     \
    cudaError_t e__ = cudaGetLastError();                                                  \
    if (e__ != cudaSuccess) {                                                              \
      b2f::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), __FILE__, __LINE__); \
      return B2F_ECUDA;                                                                    \
    }                                                                                      \
  } while (0)

// Bump allocator over one cudaMalloc'ed slab that grows (by reallocation, only between
// calls) to the high-water mark.  Every public entry point does arena.reset() first.
struct Arena {
  char *base = nullptr;
  size_t cap = 0, off = 0, need = 0;
  size_t limit = 0;       // != 0: end of the region the current carver may use (features.cu gives each detector its own)
  bool overflow = false;
  void reset() { off = 0; need = 0; limit = 0; overflow = false; }
  void region(size_t begin, size_t end) { off = begin; limit = end; }
  template <typename T> T *get(size_t n) {
    size_t bytes = (n * sizeof(T) + 255) & ~size_t(255);
    need += bytes;
    if (off + bytes > (limit ? limit : cap)) { overflow = true; return nullptr; }
    T *p = reinterpret_cast<T *>(base + off);
    off += bytes;
    return p;
  }
};

}  // namespace b2f

struct b2f_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  // The scratch arena (and the lazily built tables) are shared by every call on this context; a caller may pass its own
  // stream to the *_dev entry points.  last_stream is the stream the previous call's work was enqueued on: a call on a
  // different stream first waits for it (stream_handoff), so scratch still in flight is never overwritten.
  cudaStream_t last_stream = nullptr, pending_stream = nullptr;
  cudaEvent_t handoff_event = nullptr;
  b2f::Arena arena;       // device scratch
  void *pinned = nullptr; // pinned host staging
  size_t pinned_cap = 0;
  void *pinned_aux[3] = {nullptr, nullptr, nullptr};   // further pinned blocks with their own lifetimes (surf.cu: key staging of the two chunks in flight, counters)
  size_t pinned_aux_cap[3] = {0, 0, 0};
  long long launches = 0;
  void *canny_stats = nullptr;    // device counter (canny.cu): pixels decided by the exact fp64 tier since the context was created
  void *harris_stats = nullptr;   // device PatchStats (harris.cu): certification counters since the context was created
  void *surf_gauss = nullptr; // 109 Gaussian weights of the SURF orientation samples (surf.cu), built on first use
  void *fhog_lut = nullptr;   // 511x511 orientation-snap table (fhog.cu), built on first use
  void *nlmeans_lut = nullptr;   // 30000-entry exp(-x) table of NL-means (nlmeans.cu), uploaded on first use
  // FHOG vote tables of the last geometry (fhog.cu): one device block, rebuilt when (rows, cols, cell) changes
  void *fhog_tab = nullptr;
  size_t fhog_tab_cap = 0;
  int fhog_tab_key[3] = {0, 0, 0};
  int fhog_tab_kw = 0;
  // chunked host batches (*_batch): copy-in / copy-out streams beside `stream`, and their events
  size_t chunk_bytes = (size_t)48 << 20;   // input bytes per chunk (b2f_set_chunk_bytes, B2F_CHUNK_BYTES); composite end to end on an H100 SXM (700 W): 24 / 48 / 96 MiB 13.5 / 13.1-13.2 / 11.6 Gpixel/s
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaStream_t s_aux[2] = {nullptr, nullptr};   // the combined batch (features.cu) runs its three detectors side by side: context stream + these two
  std::vector<cudaEvent_t> events;
};

namespace b2f {
// Make sure the device scratch arena holds at least `bytes` (grows by reallocation; synchronises
// the context stream first) and rewind it.  Every public entry point calls this once with an
// upper bound of its scratch need, then carves buffers with ctx->arena.get<T>(n).
int arena_reserve(b2f_ctx *ctx, size_t bytes);
int pinned_reserve(b2f_ctx *ctx, size_t bytes);
int pinned_reserve_aux(b2f_ctx *ctx, int which, size_t bytes);   // grows block `which` only; the caller knows nothing reads it any more
// Host batches are cut into chunks of frames so that the upload of chunk c+1, the kernels of chunk c and
// the download of chunk c-1 overlap (three streams, events between them).  pipe_prepare makes sure the two
// copy streams and `n_events` events exist and orders the copy-in stream behind whatever the context
// stream still has in flight.
// Resolve the stream of a call (NULL = the context's own) and order it behind the previous call's stream when they differ.
int stream_handoff(b2f_ctx *ctx, void *user_stream, cudaStream_t *out);
int pipe_prepare(b2f_ctx *ctx, int n_events);
int pipe_drain(b2f_ctx *ctx);                       // wait for all three streams (also used on error paths)
// The host-batch pipeline of Harris, Canny and FHOG (features.cu), for any subset of them: hp = NULL, cp = NULL or
// cell_size = 0 skips a detector.  channels = 3: interleaved RGB frames (grey derived on the device); 1: grey frames
// (no FHOG).  `who` names the public entry point in error messages.
int features_batch(const char *who, b2f_ctx *ctx, const uint8_t *frames, int channels, int n_frames, int rows, int cols,
                   const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                   const b2f_canny_params *cp, uint8_t *edges, int *nonzero, int cell_size, int frp, int fcp, float *hog);
inline int frames_per_chunk(const b2f_ctx *ctx, size_t frame_bytes, int n_frames) {
  const size_t target = ctx->chunk_bytes;
  size_t c = target / (frame_bytes ? frame_bytes : 1);
  if (c < 1) c = 1;
  return c > (size_t)n_frames ? n_frames : (int)c;
}
#define B2F_ARENA_CHECK(ctx)                                                                \
  do {                                                                                     \
    if ((ctx)->arena.overflow) {                                                           \
      b2f::set_error("internal: scratch arena under-reserved (%zu needed, %zu held) at %s:%d", \
                     (ctx)->arena.need, (ctx)->arena.cap, __FILE__, __LINE__);            \
      return B2F_ENOMEM;                                                                   \
    }                                                                                      \
  } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
static inline size_t align256(size_t b) { return (b + 255) & ~size_t(255); }
}  // namespace b2f
