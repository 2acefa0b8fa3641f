// ctx.cu — lifecycle of a libb200feat context: CUDA device selection, the launch stream, the
// device scratch arena and the pinned staging buffer.  No CPU fallback exists anywhere in this
// library: b2f_init fails when no usable sm_90 device is present.
#include "common.cuh"
#include <cstdarg>

namespace b2f {
static thread_local char g_err[512] = "";

void set_error(const char *fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int order_behind_last(b2f_ctx *ctx, cudaStream_t st) {
  if (ctx->last_stream && ctx->last_stream != st) {
    if (!ctx->handoff_event) B2F_CUDA(cudaEventCreateWithFlags(&ctx->handoff_event, cudaEventDisableTiming));
    B2F_CUDA(cudaEventRecord(ctx->handoff_event, ctx->last_stream));
    B2F_CUDA(cudaStreamWaitEvent(st, ctx->handoff_event, 0));
  }
  ctx->last_stream = st;
  return B2F_OK;
}

int arena_reserve(b2f_ctx *ctx, size_t bytes) {
  // The arena is about to be rewound: whatever stream this call runs on (the one a *_dev entry point announced through
  // stream_handoff, else the context's own, as all host / batch forms use) must run behind the previous call's stream.
  cudaStream_t target = ctx->pending_stream ? ctx->pending_stream : ctx->stream;
  ctx->pending_stream = nullptr;
  int hrc = order_behind_last(ctx, target);
  if (hrc != B2F_OK) return hrc;
  ctx->arena.reset();
  if (bytes <= ctx->arena.cap) return B2F_OK;
  size_t want = bytes + (bytes >> 4) + (1u << 20);
  B2F_CUDA(cudaStreamSynchronize(ctx->stream));
  if (ctx->arena.base) B2F_CUDA(cudaFree(ctx->arena.base));
  ctx->arena.base = nullptr;
  ctx->arena.cap = 0;
  void *p = nullptr;
  cudaError_t e = cudaMalloc(&p, want);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_error("cudaMalloc(%zu bytes of scratch) failed: %s", want, cudaGetErrorString(e));
    return B2F_ENOMEM;
  }
  ctx->arena.base = static_cast<char *>(p);
  ctx->arena.cap = want;
  return B2F_OK;
}

int pinned_reserve(b2f_ctx *ctx, size_t bytes) {
  if (bytes <= ctx->pinned_cap) return B2F_OK;
  B2F_CUDA(cudaStreamSynchronize(ctx->stream));
  if (ctx->pinned) B2F_CUDA(cudaFreeHost(ctx->pinned));
  ctx->pinned = nullptr;
  ctx->pinned_cap = 0;
  void *p = nullptr;
  cudaError_t e = cudaMallocHost(&p, bytes);
  if (e != cudaSuccess) {
    set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return B2F_ENOMEM;
  }
  ctx->pinned = p;
  ctx->pinned_cap = bytes;
  return B2F_OK;
}

int pinned_reserve_aux(b2f_ctx *ctx, int which, size_t bytes) {
  if (bytes <= ctx->pinned_aux_cap[which]) return B2F_OK;
  if (ctx->pinned_aux[which]) B2F_CUDA(cudaFreeHost(ctx->pinned_aux[which]));
  ctx->pinned_aux[which] = nullptr;
  ctx->pinned_aux_cap[which] = 0;
  bytes += bytes / 4 + 4096;          // headroom: the next chunk rarely needs a new block
  void *p = nullptr;
  cudaError_t e = cudaMallocHost(&p, bytes);
  if (e != cudaSuccess) {
    set_error("cudaMallocHost(%zu) failed: %s", bytes, cudaGetErrorString(e));
    return B2F_ENOMEM;
  }
  ctx->pinned_aux[which] = p;
  ctx->pinned_aux_cap[which] = bytes;
  return B2F_OK;
}

int stream_handoff(b2f_ctx *ctx, void *user_stream, cudaStream_t *out) {
  cudaStream_t st = user_stream ? (cudaStream_t)user_stream : ctx->stream;
  *out = st;
  ctx->pending_stream = st;
  return order_behind_last(ctx, st);
}

int pipe_prepare(b2f_ctx *ctx, int n_events) {
  if (!ctx->s_in) B2F_CUDA(cudaStreamCreateWithFlags(&ctx->s_in, cudaStreamNonBlocking));
  if (!ctx->s_out) B2F_CUDA(cudaStreamCreateWithFlags(&ctx->s_out, cudaStreamNonBlocking));
  n_events += 1;
  while ((int)ctx->events.size() < n_events) {
    cudaEvent_t e;
    B2F_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    ctx->events.push_back(e);
  }
  cudaEvent_t e0 = ctx->events[n_events - 1];
  B2F_CUDA(cudaEventRecord(e0, ctx->stream));
  B2F_CUDA(cudaStreamWaitEvent(ctx->s_in, e0, 0));
  return B2F_OK;
}

int pipe_drain(b2f_ctx *ctx) {
  cudaError_t a = ctx->s_in ? cudaStreamSynchronize(ctx->s_in) : cudaSuccess;
  cudaError_t b = cudaStreamSynchronize(ctx->stream);
  cudaError_t c = cudaSuccess;
  for (cudaStream_t s : ctx->s_aux)
    if (s) { cudaError_t x = cudaStreamSynchronize(s); if (c == cudaSuccess) c = x; }
  if (ctx->s_out) { cudaError_t x = cudaStreamSynchronize(ctx->s_out); if (c == cudaSuccess) c = x; }
  cudaError_t e = a != cudaSuccess ? a : (b != cudaSuccess ? b : c);
  if (e != cudaSuccess) { cudaGetLastError(); set_error("CUDA error while draining a batch: %s", cudaGetErrorString(e)); return B2F_ECUDA; }
  return B2F_OK;
}
}  // namespace b2f

extern "C" {

const char *b2f_last_error(void) { return b2f::g_err; }
const char *b2f_version(void) { return "b200feat 0.1 (sm_90a)"; }

int b2f_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int b2f_init(int device, b2f_ctx **out) {
  if (!out) { b2f::set_error("b2f_init: ctx pointer is NULL"); return B2F_EINVAL; }
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0) {
    b2f::set_error("b2f_init: no CUDA device available (%s); this library has no CPU path",
                   e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    cudaGetLastError();
    return B2F_ECUDA;
  }
  if (device < 0 || device >= n) { b2f::set_error("b2f_init: device %d out of range [0,%d)", device, n); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  B2F_CUDA(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    b2f::set_error("b2f_init: device %d is sm_%d%d; this build contains sm_90a code only", device, prop.major, prop.minor);
    return B2F_EUNSUP;
  }
  b2f_ctx *c = new b2f_ctx();
  c->device = device;
  if (const char *cb = getenv("B2F_CHUNK_BYTES")) { const long long v = atoll(cb); if (v > 0) c->chunk_bytes = (size_t)v; }
  c->sm_count = prop.multiProcessorCount;
  e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e != cudaSuccess) { b2f::set_error("cudaStreamCreate: %s", cudaGetErrorString(e)); delete c; return B2F_ECUDA; }
  *out = c;
  return B2F_OK;
}

void b2f_shutdown(b2f_ctx *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  cudaStreamSynchronize(c->stream);
  if (c->arena.base) cudaFree(c->arena.base);
  if (c->pinned) cudaFreeHost(c->pinned);
  for (void *q : c->pinned_aux)
    if (q) cudaFreeHost(q);
  if (c->handoff_event) cudaEventDestroy(c->handoff_event);
  if (c->canny_stats) cudaFree(c->canny_stats);
  if (c->harris_stats) cudaFree(c->harris_stats);
  if (c->surf_gauss) cudaFree(c->surf_gauss);
  if (c->fhog_lut) cudaFree(c->fhog_lut);
  if (c->nlmeans_lut) cudaFree(c->nlmeans_lut);
  if (c->fhog_tab) cudaFree(c->fhog_tab);
  if (c->s_in) { cudaStreamSynchronize(c->s_in); cudaStreamDestroy(c->s_in); }
  if (c->s_out) { cudaStreamSynchronize(c->s_out); cudaStreamDestroy(c->s_out); }
  for (cudaStream_t s : c->s_aux)
    if (s) { cudaStreamSynchronize(s); cudaStreamDestroy(s); }
  for (cudaEvent_t e : c->events) cudaEventDestroy(e);
  cudaStreamDestroy(c->stream);
  delete c;
}

void b2f_free(void *p) { free(p); }
int b2f_set_chunk_bytes(b2f_ctx *c, size_t bytes) {
  if (!c || bytes == 0) { b2f::set_error("b2f_set_chunk_bytes: bad argument"); return B2F_EINVAL; }
  c->chunk_bytes = bytes;
  return B2F_OK;
}
void *b2f_stream(b2f_ctx *c) { return c ? (void *)c->stream : nullptr; }
long long b2f_launch_count(b2f_ctx *c) { return c ? c->launches : 0; }

}  // extern "C"
