// lsd.cu — front end of image.LineSegmentDetector (SURVEY.md 8f rank 2) on the device:
//   gaussian_sampler  lsd.c:603-720   Gaussian sub-sampling to `scale` (0.8): one kernel per axis, each output sample has
//                                     its own 2h+1 taps centred on sample/scale, symmetric boundary, double accumulation
//   ll_angle          lsd.c:744-880   2x2 gradient, modulus, level-line angle atan2(gx, -gy) (NOTDEF below the threshold),
//                                     and the list of pixels pseudo-ordered by decreasing modulus (n_bins buckets,
//                                     inside a bucket in the reference's visiting order: x outer, y inner)
// The region grower that consumes these stays sequential on the CPU (lsd.c:region_grow); it needs the angle and
// modulus planes and the ordered list, which is what comes back.  modgrad, the bucket of every pixel and the list
// order are bit-identical to the reference (IEEE double, one rounding per operation, taps computed on the host with
// the same libm exp); the angles go through CUDA's atan2 (<= 2 ulp) where the reference calls libm's: the decision
// `norm <= threshold` -> NOTDEF is made on the bit-exact modulus, so the NOTDEF pattern is identical and the defined
// angles agree to ~1e-15.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <vector>

namespace b2f {

constexpr double LSD_NOTDEF = -1024.0;      // lsd.c:103
constexpr int LSD_MAX_TAPS = 64, LSD_CHUNK = 2048, LSD_MAX_BINS = 4096;

__device__ __forceinline__ int lsd_mirror(int j, int n) {      // lsd.c:667-670
  const int n2 = 2 * n;
  while (j < 0) j += n2;
  while (j >= n2) j -= n2;
  return j >= n ? n2 - 1 - j : j;
}

// x axis: aux[x + y*N] = sum_i in[mirror(cx[x]-h+i) + y*X] * kx[x][i]   (lsd.c:645-677)
template <typename T>
__global__ void __launch_bounds__(256)
lsd_sample_x_kernel(const T *__restrict__ in, double *__restrict__ aux, const double *__restrict__ kx, const int *__restrict__ cx,
                    int X, int Y, int N, int h) {
  const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  if (x >= N) return;
  const T *row = in + ((size_t)blockIdx.z * Y + y) * X;
  const double *k = kx + (size_t)x * (2 * h + 1);
  const int c = cx[x] - h;
  double s = 0.0;
  for (int i = 0; i <= 2 * h; i++) s = __dadd_rn(s, __dmul_rn((double)row[lsd_mirror(c + i, X)], k[i]));
  aux[((size_t)blockIdx.z * Y + y) * N + x] = s;
}

// y axis: out[x + y*N] = sum_i aux[x + mirror(cy[y]-h+i)*N] * ky[y][i]   (lsd.c:680-712)
__global__ void __launch_bounds__(256)
lsd_sample_y_kernel(const double *__restrict__ aux, double *__restrict__ out, const double *__restrict__ ky, const int *__restrict__ cy,
                    int Y, int N, int M, int h) {
  const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  if (x >= N) return;
  const double *src = aux + (size_t)blockIdx.z * Y * N + x;
  const double *k = ky + (size_t)y * (2 * h + 1);
  const int c = cy[y] - h;
  double s = 0.0;
  for (int i = 0; i <= 2 * h; i++) s = __dadd_rn(s, __dmul_rn(__ldg(src + (size_t)lsd_mirror(c + i, Y) * N), k[i]));
  out[((size_t)blockIdx.z * M + y) * N + x] = s;
}

// gradient, modulus, angle (lsd.c:796-834) + the frame's largest defined modulus (non-negative doubles order like their bits)
__global__ void __launch_bounds__(256)
lsd_gradient_kernel(const double *__restrict__ in, double *__restrict__ angles, double *__restrict__ modgrad,
                    unsigned long long *__restrict__ max_bits, int N, int M, double threshold) {
  const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y;
  const size_t base = (size_t)blockIdx.z * N * M;
  double mx = 0.0;
  if (x < N) {
    const size_t a = base + (size_t)y * N + x;
    if (x == N - 1 || y == M - 1) {
      angles[a] = LSD_NOTDEF;               // 'undefined' on the down and right boundaries (:790-792)
      modgrad[a] = 0.0;                     // (uninitialised in the reference; never read by it)
    } else {
      const double A = in[a], B = in[a + 1], Cc = in[a + N], D = in[a + N + 1];
      const double com1 = __dsub_rn(D, A), com2 = __dsub_rn(B, Cc);
      const double gx = __dadd_rn(com1, com2), gy = __dsub_rn(com1, com2);
      const double norm = __dsqrt_rn(__ddiv_rn(__dadd_rn(__dmul_rn(gx, gx), __dmul_rn(gy, gy)), 4.0));
      modgrad[a] = norm;
      if (norm <= threshold) angles[a] = LSD_NOTDEF;
      else { angles[a] = atan2(gx, -gy); mx = norm; }
    }
  }
  for (int o = 16; o; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if ((threadIdx.x & 31) == 0 && mx > 0.0) atomicMax(max_bits + blockIdx.z, (unsigned long long)__double_as_longlong(mx));
}

// The ordered list is a stable counting sort of the (N-1)(M-1) gradient pixels, visited x outer / y inner, by bucket
// (highest first).  Sequence position s <-> (x = s / (M-1), y = s % (M-1)).
// A frame without a defined angle keeps max_grad == 0, and the reference's quotient is NaN (norm 0) or +inf.  Its
// (unsigned) conversion is undefined in C; the x86-64 build truncates through a signed 64-bit integer, which gives
// INT64_MIN, low 32 bits 0: every pixel lands in bucket 0 (DESIGN.md §5).  That is decided here, not left to the
// device's conversion (sm_90 gives 0x80000000 for NaN and 0xFFFFFFFF for +inf: one clamped bucket too, by accident).
__device__ __forceinline__ int lsd_bucket(double norm, double max_grad, int n_bins) {     // lsd.c:844-845
  if (!(max_grad > 0.0)) return 0;
  unsigned i = (unsigned)__ddiv_rn(__dmul_rn(norm, (double)n_bins), max_grad);
  return i >= (unsigned)n_bins ? n_bins - 1 : (int)i;
}

__global__ void __launch_bounds__(256)
lsd_bucket_hist_kernel(const double *__restrict__ modgrad, const unsigned long long *__restrict__ max_bits, int *__restrict__ counts,
                       int N, int M, int n_bins, int n_chunks) {
  extern __shared__ int hist[];
  const int chunk = blockIdx.x, f = blockIdx.y;
  for (int b = threadIdx.x; b < n_bins; b += 256) hist[b] = 0;
  __syncthreads();
  const double max_grad = __longlong_as_double((long long)max_bits[f]);
  const long long total = (long long)(N - 1) * (M - 1);
  const double *mg = modgrad + (size_t)f * N * M;
  for (int k = threadIdx.x; k < LSD_CHUNK; k += 256) {
    const long long s = (long long)chunk * LSD_CHUNK + k;
    if (s < total) {
      const int x = (int)(s / (M - 1)), y = (int)(s - (long long)x * (M - 1));
      atomicAdd(&hist[lsd_bucket(mg[(size_t)y * N + x], max_grad, n_bins)], 1);
    }
  }
  __syncthreads();
  int *dst = counts + ((size_t)f * n_chunks + chunk) * n_bins;
  for (int b = threadIdx.x; b < n_bins; b += 256) dst[b] = hist[b];
}

// per bucket: exclusive prefix over the chunks (in place); totals[f][b] = size of the bucket
__global__ void lsd_bucket_scan_chunks_kernel(int *__restrict__ counts, int *__restrict__ totals, int n_bins, int n_chunks) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x, f = blockIdx.y;
  if (b >= n_bins) return;
  int *c = counts + (size_t)f * n_chunks * n_bins + b;
  int run = 0;
  for (int k = 0; k < n_chunks; k++) { const int v = c[(size_t)k * n_bins]; c[(size_t)k * n_bins] = run; run += v; }
  totals[(size_t)f * n_bins + b] = run;
}

// one CTA per frame: start of every bucket in the list, highest bucket first (lsd.c:861-873), in place
__global__ void __launch_bounds__(1024)
lsd_bucket_starts_kernel(int *__restrict__ totals, int n_bins) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  int *t = totals + (size_t)blockIdx.x * n_bins;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_bins; base += 1024) {
    const int j = base + threadIdx.x;                 // j-th bucket from the top
    const int b = n_bins - 1 - j;
    const int v = j < n_bins ? t[b] : 0;
    int incl = v;
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += u; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = warp_tot[lane], wi = w;
      for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += u; }
      warp_tot[lane] = wi - w;
    }
    __syncthreads();
    const int excl = carry + warp_tot[warp] + incl - v;
    if (j < n_bins) t[b] = excl;
    __syncthreads();
    if (threadIdx.x == 1023) carry = excl + v;
    __syncthreads();
  }
}

// one CTA per chunk: stable scatter.  The chunk is walked 256 elements at a time, warp after warp, so that elements of
// the same bucket keep their sequence order: rank inside a warp from __match_any_sync, across warps / rounds through
// the shared running position of the bucket.
__global__ void __launch_bounds__(256)
lsd_bucket_scatter_kernel(const double *__restrict__ modgrad, const unsigned long long *__restrict__ max_bits,
                          const int *__restrict__ counts, const int *__restrict__ starts, int *__restrict__ list,
                          int N, int M, int n_bins, int n_chunks) {
  extern __shared__ int pos[];
  const int chunk = blockIdx.x, f = blockIdx.y;
  const int *cpre = counts + ((size_t)f * n_chunks + chunk) * n_bins;
  const int *st = starts + (size_t)f * n_bins;
  for (int b = threadIdx.x; b < n_bins; b += 256) pos[b] = st[b] + cpre[b];
  __syncthreads();
  const double max_grad = __longlong_as_double((long long)max_bits[f]);
  const long long total = (long long)(N - 1) * (M - 1);
  const double *mg = modgrad + (size_t)f * N * M;
  int *out = list + (size_t)f * total;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int round = 0; round < LSD_CHUNK / 256; round++) {
    const long long s = (long long)chunk * LSD_CHUNK + round * 256 + threadIdx.x;
    const bool valid = s < total;
    int x = 0, y = 0, b = 0;
    if (valid) {
      x = (int)(s / (M - 1)); y = (int)(s - (long long)x * (M - 1));
      b = lsd_bucket(mg[(size_t)y * N + x], max_grad, n_bins);
    }
    for (int w = 0; w < 8; w++) {
      if (warp == w) {
        const unsigned act = __ballot_sync(0xffffffffu, valid);
        if (valid) {
          const unsigned same = __match_any_sync(act, b);
          const int rank = __popc(same & ((1u << lane) - 1u));
          const int first = pos[b];
          __syncwarp(act);
          if (rank == 0) pos[b] = first + __popc(same);
          out[first + rank] = x + y * N;
        }
      }
      __syncthreads();
    }
  }
}

struct LsdPlan {
  int N, M, h, n;
  double sigma;
  std::vector<double> kx, ky;
  std::vector<int> cx, cy;
};

static void lsd_kernel_row(double *k, int dim, double sigma, double mean) {      // gaussian_kernel, lsd.c:540-561
  double sum = 0.0;
  for (int i = 0; i < dim; i++) {
    const double v = ((double)i - mean) / sigma;
    k[i] = exp(-0.5 * v * v);
    sum += k[i];
  }
  if (sum >= 0.0) for (int i = 0; i < dim; i++) k[i] /= sum;
}

static int lsd_plan(int X, int Y, double scale, double sigma_scale, LsdPlan &p) {
  if (!(scale > 0.0) || !(sigma_scale > 0.0)) { set_error("lsd: scale and sigma_scale must be positive"); return B2F_EINVAL; }
  p.N = (int)(unsigned)ceil(X * scale);                     // lsd.c:623-624
  p.M = (int)(unsigned)ceil(Y * scale);
  p.sigma = scale < 1.0 ? sigma_scale / scale : sigma_scale;
  p.h = (int)(unsigned)ceil(p.sigma * sqrt(2.0 * 3.0 * log(10.0)));
  p.n = 1 + 2 * p.h;
  if (p.n > LSD_MAX_TAPS) { set_error("lsd: kernel of %d taps exceeds %d", p.n, LSD_MAX_TAPS); return B2F_EUNSUP; }
  if (p.N < 2 || p.M < 2 || (long long)p.N * p.M >= (1ll << 31)) { set_error("lsd: scaled size %dx%d unsupported", p.N, p.M); return B2F_EUNSUP; }
  auto axis = [&](int n_out, std::vector<double> &k, std::vector<int> &c) {   // lsd.c:655-661 / :690-696
    k.resize((size_t)n_out * p.n); c.resize(n_out);
    for (int u = 0; u < n_out; u++) {
      const double uu = (double)u / scale;
      const int uc = (int)floor(uu + 0.5);
      lsd_kernel_row(&k[(size_t)u * p.n], p.n, p.sigma, (double)p.h + uu - (double)uc);
      c[u] = uc;
    }
  };
  axis(p.N, p.kx, p.cx);
  axis(p.M, p.ky, p.cy);
  return B2F_OK;
}

size_t lsd_scratch_bytes(int n_frames, int X, int Y, int N, int M, int n_bins) {
  const long long total = (long long)(N - 1) * (M - 1);
  const int n_chunks = (int)((total + LSD_CHUNK - 1) / LSD_CHUNK);
  size_t b = align256((size_t)n_frames * N * Y * 8) + align256((size_t)n_frames * N * M * 8);             // aux, scaled
  b += align256((size_t)(N + M) * LSD_MAX_TAPS * 8) + align256((size_t)(N + M) * 4) * 2;                 // taps, centres
  b += align256((size_t)n_frames * n_chunks * n_bins * 4) + align256((size_t)n_frames * n_bins * 4) + align256((size_t)n_frames * 8);
  return b + 8192;
}

// frames on the device -> angles, modgrad [n][M][N], list [n][(N-1)(M-1)]; d_scaled optional
int lsd_front_device(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int X, int Y, const LsdPlan &p, double threshold,
                     int n_bins, double *d_angles, double *d_modgrad, int *d_list, double *d_scaled, cudaStream_t st) {
  const int N = p.N, M = p.M;
  const long long total = (long long)(N - 1) * (M - 1);
  const int n_chunks = (int)((total + LSD_CHUNK - 1) / LSD_CHUNK);
  double *aux = ctx->arena.get<double>((size_t)n_frames * N * Y);
  double *scaled = d_scaled ? d_scaled : ctx->arena.get<double>((size_t)n_frames * N * M);
  double *kx = ctx->arena.get<double>(p.kx.size()), *ky = ctx->arena.get<double>(p.ky.size());
  int *cx = ctx->arena.get<int>(N), *cy = ctx->arena.get<int>(M);
  int *counts = ctx->arena.get<int>((size_t)n_frames * n_chunks * n_bins);
  int *totals = ctx->arena.get<int>((size_t)n_frames * n_bins);
  unsigned long long *maxb = ctx->arena.get<unsigned long long>(n_frames);
  B2F_ARENA_CHECK(ctx);
  // the tables are small (tens of KB); pageable-source copies are staged by the runtime before the call returns
  B2F_CUDA(cudaMemcpyAsync(kx, p.kx.data(), p.kx.size() * 8, cudaMemcpyHostToDevice, st));
  B2F_CUDA(cudaMemcpyAsync(ky, p.ky.data(), p.ky.size() * 8, cudaMemcpyHostToDevice, st));
  B2F_CUDA(cudaMemcpyAsync(cx, p.cx.data(), (size_t)N * 4, cudaMemcpyHostToDevice, st));
  B2F_CUDA(cudaMemcpyAsync(cy, p.cy.data(), (size_t)M * 4, cudaMemcpyHostToDevice, st));
  B2F_CUDA(cudaMemsetAsync(maxb, 0, sizeof(unsigned long long) * n_frames, st));
  if (u8) lsd_sample_x_kernel<unsigned char><<<dim3(ceil_div(N, 256), Y, n_frames), 256, 0, st>>>(static_cast<const unsigned char *>(d_frames), aux, kx, cx, X, Y, N, p.h);
  else lsd_sample_x_kernel<double><<<dim3(ceil_div(N, 256), Y, n_frames), 256, 0, st>>>(static_cast<const double *>(d_frames), aux, kx, cx, X, Y, N, p.h);
  B2F_LAUNCH_CHECK(ctx);
  lsd_sample_y_kernel<<<dim3(ceil_div(N, 256), M, n_frames), 256, 0, st>>>(aux, scaled, ky, cy, Y, N, M, p.h);
  B2F_LAUNCH_CHECK(ctx);
  lsd_gradient_kernel<<<dim3(ceil_div(N, 256), M, n_frames), 256, 0, st>>>(scaled, d_angles, d_modgrad, maxb, N, M, threshold);
  B2F_LAUNCH_CHECK(ctx);
  const size_t sm = sizeof(int) * n_bins;
  lsd_bucket_hist_kernel<<<dim3(n_chunks, n_frames), 256, sm, st>>>(d_modgrad, maxb, counts, N, M, n_bins, n_chunks);
  B2F_LAUNCH_CHECK(ctx);
  lsd_bucket_scan_chunks_kernel<<<dim3(ceil_div(n_bins, 128), n_frames), 128, 0, st>>>(counts, totals, n_bins, n_chunks);
  B2F_LAUNCH_CHECK(ctx);
  lsd_bucket_starts_kernel<<<n_frames, 1024, 0, st>>>(totals, n_bins);
  B2F_LAUNCH_CHECK(ctx);
  lsd_bucket_scatter_kernel<<<dim3(n_chunks, n_frames), 256, sm, st>>>(d_modgrad, maxb, counts, totals, d_list, N, M, n_bins, n_chunks);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

static int lsd_check(const char *who, int X, int Y, double quant, double ang_th, int n_bins) {
  if (X <= 0 || Y <= 0) { set_error("%s: invalid image input", who); return B2F_EINVAL; }
  if (quant < 0.0 || ang_th <= 0.0 || ang_th >= 180.0) { set_error("%s: quant / ang_th out of range (lsd.c:2437-2440)", who); return B2F_EINVAL; }
  if (n_bins <= 0 || n_bins > LSD_MAX_BINS) { set_error("%s: n_bins must be in 1..%d", who, LSD_MAX_BINS); return B2F_EINVAL; }
  return B2F_OK;
}

static double lsd_rho(double quant, double ang_th) { return quant / sin(M_PI * ang_th / 180.0); }   // lsd.c:2449-2451

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_lsd_front_size(int X, int Y, double scale, int *N, int *M) {
  if (!N || !M || X <= 0 || Y <= 0 || !(scale > 0.0)) { set_error("b2f_lsd_front_size: bad argument"); return B2F_EINVAL; }
  *N = (int)(unsigned)ceil(X * scale);
  *M = (int)(unsigned)ceil(Y * scale);
  return B2F_OK;
}

int b2f_lsd_front_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int X, int Y, double scale, double sigma_scale,
                      double quant, double ang_th, int n_bins, double *d_angles, double *d_modgrad, int *d_list, double *d_scaled,
                      void *stream) {
  if (!ctx || !d_frames || !d_angles || !d_modgrad || !d_list || n_frames <= 0) { set_error("b2f_lsd_front_dev: bad argument"); return B2F_EINVAL; }
  int rc = lsd_check("b2f_lsd_front_dev", X, Y, quant, ang_th, n_bins);
  if (rc != B2F_OK) return rc;
  if (scale == 1.0) { set_error("b2f_lsd_front_dev: scale 1 (no sampling) is served by b2f_lsd_front_host only"); return B2F_EUNSUP; }
  LsdPlan p;
  if ((rc = lsd_plan(X, Y, scale, sigma_scale, p)) != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  { int hrc = stream_handoff(ctx, stream, &st); if (hrc != B2F_OK) return hrc; }
  if ((rc = arena_reserve(ctx, lsd_scratch_bytes(n_frames, X, Y, p.N, p.M, n_bins))) != B2F_OK) return rc;
  // (the plan's pageable tables are staged by cudaMemcpyAsync before it returns, so `p` may go out of scope)
  return lsd_front_device(ctx, d_frames, is_u8 != 0, n_frames, X, Y, p, lsd_rho(quant, ang_th), n_bins, d_angles, d_modgrad, d_list, d_scaled, st);
}

// one image of doubles in host memory (what detect_line_segments receives, line_segment_detector.cpp:8-33)
int b2f_lsd_front_host(b2f_ctx *ctx, const double *image, int X, int Y, double scale, double sigma_scale, double quant, double ang_th,
                       int n_bins, double *angles, double *modgrad, int *list, int *list_len, double *scaled) {
  if (!ctx || !image || !angles || !modgrad || !list || !list_len) { set_error("b2f_lsd_front_host: bad argument"); return B2F_EINVAL; }
  int rc = lsd_check("b2f_lsd_front_host", X, Y, quant, ang_th, n_bins);
  if (rc != B2F_OK) return rc;
  if (scale == 1.0) { set_error("b2f_lsd_front_host: scale must differ from 1 (the reference skips the sampler then; not served yet)"); return B2F_EUNSUP; }
  LsdPlan p;
  if ((rc = lsd_plan(X, Y, scale, sigma_scale, p)) != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st = ctx->stream;
  const size_t in_px = (size_t)X * Y, out_px = (size_t)p.N * p.M, total = (size_t)(p.N - 1) * (p.M - 1);
  rc = arena_reserve(ctx, lsd_scratch_bytes(1, X, Y, p.N, p.M, n_bins) + align256(in_px * 8) + 3 * align256(out_px * 8) + align256(total * 4));
  if (rc != B2F_OK) return rc;
  double *d_img = ctx->arena.get<double>(in_px), *d_ang = ctx->arena.get<double>(out_px), *d_mod = ctx->arena.get<double>(out_px),
         *d_sc = ctx->arena.get<double>(out_px);
  int *d_list = ctx->arena.get<int>(total);
  B2F_ARENA_CHECK(ctx);
  B2F_CUDA(cudaMemcpyAsync(d_img, image, in_px * 8, cudaMemcpyHostToDevice, st));
  rc = lsd_front_device(ctx, d_img, false, 1, X, Y, p, lsd_rho(quant, ang_th), n_bins, d_ang, d_mod, d_list, d_sc, st);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaMemcpyAsync(angles, d_ang, out_px * 8, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaMemcpyAsync(modgrad, d_mod, out_px * 8, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaMemcpyAsync(list, d_list, total * 4, cudaMemcpyDeviceToHost, st));
  if (scaled) B2F_CUDA(cudaMemcpyAsync(scaled, d_sc, out_px * 8, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  *list_len = (int)total;
  return B2F_OK;
}

}  // extern "C"
