// harris_api.cu — C ABI of the Harris path (include/b2f.h) and the tail of the detector: output
// selection, sub-pixel refinement and the scale-stability check (SURVEY.md 8a row H7: harris.cpp:263-381,
// :443-465, :554-608; interpolation.cpp).  These touch a few thousand corners per frame (<1 % of the
// reference's time).  The float expressions are the reference's (the results have to be bit-identical, so
// each rounding step is dictated: same operand order, same float/double promotions, no FMA contraction —
// this file is compiled with -ffp-contract=off), the organisation is ours: corners carry the index of their
// device record so that the 3x3 neighbourhoods computed on the device (exact patches) follow them through
// the selection.
#include "harris_host.h"
#include <algorithm>
#include <cmath>
#include <vector>

namespace b2f {

struct Corner { float x, y, R; int rec; };                     // rec = index of the device record (3x3 patch)
static inline bool operator<(const Corner &a, const Corner &b) { return a.R > b.R; }   // strongest first (harris.cpp:29-36)

static void keep_strongest(std::vector<Corner> &c, int N) {     // sort, then truncate to N (std::sort: same
  std::sort(c.begin(), c.end());                                // comparison sequence as the reference's, hence the
  if (N >= 0 && N < (int)c.size()) c.resize(N);                 // same order among equal strengths)
}

// harris.cpp:272-331: 0 all, 1 all sorted, 2 N strongest, 3 N strongest spread over a cells x cells grid
static void select_output_corners(std::vector<Corner> &c, int strategy, int cells, int N, int nx, int ny) {
  if (strategy == 1) { keep_strongest(c, -1); return; }
  if (strategy == 2) { keep_strongest(c, N); return; }
  if (strategy != 3) return;
  const int gx = std::min(cells, nx), gy = std::min(cells, ny), nbins = gx * gy;
  const int per_bin = std::max(N / nbins, 1);
  const float wx = (float)nx / gx, wy = (float)ny / gy;         // bin extents, float like the reference
  std::vector<std::vector<Corner>> bins(nbins);
  for (const Corner &k : c) {
    const int bx = (float)k.x / wx, by = (float)k.y / wy;       // float division, truncated (harris.cpp:303-304)
    bins[(int)(by * gx + bx)].push_back(k);
  }
  c.clear();
  for (std::vector<Corner> &b : bins) {
    std::sort(b.begin(), b.end());
    c.insert(c.end(), b.begin(), b.begin() + std::min(b.size(), (size_t)per_bin));
  }
  keep_strongest(c, N);
}

// interpolation.cpp:27-54 — maximum of the quadratic fitted to the 3x3 neighbourhood M (row-major)
static bool refine_quadratic(const float *M, float &x, float &y, float &Mo) {
  const float c = M[4], l = M[3], r = M[5], u = M[1], d = M[7];
  float fx = 0.5 * (r - l);
  float fy = 0.5 * (d - u);
  float fxx = (r - 2 * c + l);
  float fyy = (d - 2 * c + u);
  float fxy = 0.25 * (M[0] - M[2] - M[6] + M[8]);
  float det = fxx * fyy - fxy * fxy;
  if (det * det < 1E-6) return false;
  float dx = (fyy * fx - fxy * fy) / det;
  float dy = (fxx * fy - fxy * fx) / det;
  x -= dx; y -= dy;
  Mo = c + fx * dx + fy * dy + 0.5 * (fxx * dx * dx + 2 * dx * dy * fxy + fyy * dy * dy);
  return true;
}

// interpolation.cpp:62-212 — Newton iteration on the bi-quadratic (9 coefficients) through the 3x3 values
struct Biquad {
  float a[9];
  explicit Biquad(const float *M) {
    a[0] = M[4] - 0.5 * (M[1] + M[3] + M[5] + M[7]) + 0.25 * (M[0] + M[2] + M[6] + M[8]);
    a[1] = 0.5 * (M[1] - M[7]) + 0.25 * (-M[0] - M[2] + M[6] + M[8]);
    a[2] = 0.5 * (M[3] - M[5]) + 0.25 * (-M[0] + M[2] - M[6] + M[8]);
    a[3] = 0.5 * (M[3] + M[5]) - M[4];
    a[4] = 0.5 * (M[1] + M[7]) - M[4];
    a[5] = 0.25 * (M[0] - M[2] - M[6] + M[8]);
    a[6] = 0.5 * (M[5] - M[3]);
    a[7] = 0.5 * (M[7] - M[1]);
    a[8] = M[4];
  }
  void gradient(float dx, float dy, float *D) const {
    D[0] = 2 * a[0] * dx * dy * dy + 2 * a[1] * dx * dy + 2 * a[2] * dy * dy + 2 * a[3] * dx + a[5] * dy + a[6];
    D[1] = 2 * a[0] * dx * dx * dy + 2 * a[1] * dx * dx + 2 * a[2] * dx * dy + 2 * a[4] * dy + a[5] * dx + a[7];
  }
  void hessian(float dx, float dy, float *H) const {
    H[0] = 2 * a[0] * dy * dy + 2 * a[1] * dy + 2 * a[3];
    H[1] = 4 * a[0] * dx * dy + 2 * a[1] * dx + 2 * a[2] * dy + a[5];
    H[2] = 2 * a[0] * dx * dx + 2 * a[2] * dx + 2 * a[4];
  }
  float value(float dx, float dy) const {
    return a[0] * dx * dx * dy * dy + a[1] * dx * dx * dy + a[2] * dx * dy * dy + a[3] * dx * dx + a[4] * dy * dy +
           a[5] * dx * dy + a[6] * dx + a[7] * dy + a[8];
  }
};
static bool refine_quartic(const float *M, float &x, float &y, float &Mo) {
  const Biquad f(M);
  float dx = 0, dy = 0, D[2], H[3];
  const float TOL = 1E-10;
  for (int it = 0;;) {
    f.gradient(dx, dy, D);
    f.hessian(dx, dy, H);
    float det = H[0] * H[2] - H[1] * H[1];
    if (det * det < 1E-10) return false;
    float sx = (D[0] * H[2] - D[1] * H[1]) / det;
    float sy = (D[1] * H[0] - D[0] * H[1]) / det;
    dx -= sx; dy -= sy;
    if (!(D[0] * D[0] + D[1] * D[1] > TOL && ++it < 20)) break;
  }
  if (dx > 1 || dx < -1 || dy > 1 || dy < -1 || std::isnan(dx) || std::isnan(dy)) return false;
  x += dx; y += dy;
  Mo = f.value(dx, dy);
  return true;
}

// params.exact: 0 = default: certified fast path where it exists (reference-identical lists), else the staged
// exact kernels; 1 = staged exact kernels; 2 = fused fp32 response + plain NMS, uncertified (R within 1e-4).
enum { MODE_DEFAULT = 0, MODE_STAGED = 1, MODE_FAST = 2 };
static int harris_mode(const b2f_harris_params *p) { return p->exact == 1 ? MODE_STAGED : (p->exact == 2 ? MODE_FAST : MODE_DEFAULT); }
// harris_response_device's `exact` argument for a mode when the certified path does not apply
static int staged_flag(int mode) { return mode == MODE_FAST ? 0 : 1; }

size_t harris_scratch_bytes(int n_frames, int nx, int ny, const b2f_harris_params *p, int cap) {
  size_t plane = align256((size_t)nx * ny * sizeof(float)) * n_frames;
  size_t b = plane /*R*/ + 5 * plane /*exact path: I,T,A,B,C*/;
  b += align256((size_t)n_frames * ny * ceil_div(nx, 32) * 4) + align256((size_t)n_frames * ny * 4);   // mask, row offsets
  b += align256((size_t)n_frames * nx * ny);                                                          // skip mask of a rescan
  b += 3 * align256((size_t)n_frames * cap * 4) + align256(n_frames * 4) + align256((size_t)n_frames * cap * 36);
  b += harris_certified_scratch_bytes(n_frames, nx, ny, cap, true);
  if (p->gaussian != 0) {   // SII line buffers
    int nmax = nx > ny ? nx : ny;
    double sg = std::max(p->sigma_d, p->sigma_i);
    int pad = (int)(76 * (sg / (100.0 / 3.14159265358979323846)) + 0.5) + 1;
    b += align256((size_t)n_frames * nmax * (nmax + 2 * pad) * 4);
  }
  return b + (1 << 16);
}

int harris_corners_device(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny, const b2f_harris_params *p,
                          int cap, int *d_xy, float *d_strength, int *d_counts, float *d_R, cudaStream_t st) {
  const int radius = 2 * p->sigma_i + 0.5;
  if (nx < 3 || ny < 3 || ny <= 2 * radius + 1 || nx <= 2 * radius + 1) {   // harris.cpp:493, :151
    B2F_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int) * n_frames, st));
    return B2F_OK;
  }
  const int mode = harris_mode(p);
  if (mode == MODE_DEFAULT && harris_certified_supported(nx, ny, p))
    return harris_corners_certified(ctx, d_frames, u8, n_frames, nx, ny, p, cap, d_xy, d_strength, nullptr, d_counts, d_R, st);
  float *R = d_R ? d_R : ctx->arena.get<float>((size_t)nx * ny * n_frames);
  B2F_ARENA_CHECK(ctx);
  int rc = harris_response_device(ctx, d_frames, u8, n_frames, nx, ny, p, staged_flag(mode), R, st);
  if (rc != B2F_OK) return rc;
  return harris_nms_device(ctx, R, n_frames, nx, ny, p->threshold, radius, cap, d_xy, d_strength, d_counts, st);
}

// harris() for one float plane resident on the device (harris.cpp:473-546)
static int harris_one(b2f_ctx *ctx, const float *d_I, int nx, int ny, const b2f_harris_params *p, float sigma_i,
                      int mode, std::vector<Corner> &out) {
  out.clear();
  if (nx < 3 || ny < 3) return B2F_OK;                              // harris.cpp:493
  cudaStream_t st = ctx->stream;
  b2f_harris_params q = *p;
  q.sigma_i = sigma_i;
  const size_t mark = ctx->arena.off;
  const int radius = 2 * sigma_i + 0.5;                             // harris.cpp:523
  const bool nms_runs = !(ny <= 2 * radius + 1 || nx <= 2 * radius + 1);   // harris.cpp:151
  const bool subpix = q.precision == 1 || q.precision == 2;
  const int cap = (nx / 2 + 1) * (ny / 2 + 1);                      // strict local maxima cannot be denser
  float *d_R = ctx->arena.get<float>((size_t)nx * ny);
  int *d_xy = ctx->arena.get<int>(cap);
  float *d_s = ctx->arena.get<float>(cap);
  int *d_cnt = ctx->arena.get<int>(1);
  B2F_ARENA_CHECK(ctx);
  const bool certified = mode == MODE_DEFAULT && harris_certified_supported(nx, ny, &q);
  float *d_M9 = nullptr;
  int rc, n = 0;
  std::vector<int> xy;
  std::vector<float> sv, M;
  if (certified) {
    // candidates cannot be denser than one per 2x2 block either: two 8-connected pixels cannot both be within
    // the bound of being the maximum of each other's window unless their bounds overlap; cap is re-checked below
    if (subpix) d_M9 = ctx->arena.get<float>((size_t)cap * 9);
    B2F_ARENA_CHECK(ctx);
    rc = harris_corners_certified(ctx, d_I, false, 1, nx, ny, &q, cap, d_xy, d_s, d_M9, d_cnt, d_R, st);
    if (rc != B2F_OK) return rc;
  } else {
    rc = harris_response_device(ctx, d_I, false, 1, nx, ny, &q, staged_flag(mode), d_R, st);
    if (rc != B2F_OK) return rc;
    if (nms_runs && (rc = harris_nms_device(ctx, d_R, 1, nx, ny, q.threshold, radius, cap, d_xy, d_s, d_cnt, st)) != B2F_OK) return rc;
  }
  if (nms_runs) {
    B2F_CUDA(cudaMemcpyAsync(&n, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
    B2F_CUDA(cudaStreamSynchronize(st));
    if (n < 0) {                                                     // candidate records overflowed (ties over large flat areas), or a corner
                                                                     // ties its left neighbour (harris_exact_patch_kernel): staged path
      ctx->arena.off = mark;
      return harris_one(ctx, d_I, nx, ny, p, sigma_i, MODE_STAGED, out);
    }
    if (n > cap) { set_error("harris: internal corner capacity exceeded (%d > %d)", n, cap); return B2F_ECAP; }
    xy.resize(n); sv.resize(n);
    if (n) {
      B2F_CUDA(cudaMemcpyAsync(xy.data(), d_xy, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
      B2F_CUDA(cudaMemcpyAsync(sv.data(), d_s, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
      if (d_M9) { M.resize((size_t)n * 9); B2F_CUDA(cudaMemcpyAsync(M.data(), d_M9, sizeof(float) * 9 * n, cudaMemcpyDeviceToHost, st)); }
      B2F_CUDA(cudaStreamSynchronize(st));
    }
  }
  out.resize(n);
  for (int i = 0; i < n; i++) out[i] = Corner{(float)(xy[i] % nx), (float)(xy[i] / nx), sv[i], i};
  select_output_corners(out, q.strategy, q.cells, q.Nselect, nx, ny);
  if (subpix && !out.empty()) {                                      // harris.cpp:528-532, :340-381
    const int m = (int)out.size();
    if (!d_M9) {                                                     // 3x3 neighbourhoods of the selected corners from the R plane
      std::vector<int> sel(m);
      for (int i = 0; i < m; i++) { sel[i] = (int)out[i].y * nx + (int)out[i].x; out[i].rec = i; }
      int *d_sel = ctx->arena.get<int>(m);
      float *d_M = ctx->arena.get<float>((size_t)m * 9);
      B2F_ARENA_CHECK(ctx);
      M.resize((size_t)m * 9);
      B2F_CUDA(cudaMemcpyAsync(d_sel, sel.data(), sizeof(int) * m, cudaMemcpyHostToDevice, st));
      if ((rc = harris_gather3x3(ctx, d_R, d_sel, d_M, m, nx, st)) != B2F_OK) return rc;
      B2F_CUDA(cudaMemcpyAsync(M.data(), d_M, sizeof(float) * m * 9, cudaMemcpyDeviceToHost, st));
      B2F_CUDA(cudaStreamSynchronize(st));
    }
    for (Corner &c : out) {
      const float *M9 = &M[(size_t)c.rec * 9];
      if (q.precision == 1) refine_quadratic(M9, c.x, c.y, c.R);
      else refine_quartic(M9, c.x, c.y, c.R);
    }
  }
  ctx->arena.off = mark;   // release this level's scratch
  return B2F_OK;
}

// harris_scale() (harris.cpp:554-608)
static int harris_scale(b2f_ctx *ctx, const float *d_I, int nx, int ny, const b2f_harris_params *p, int Nscales,
                        float sigma_i, int mode, std::vector<Corner> &out) {
  if (Nscales <= 1 || nx <= 64 || ny <= 64) return harris_one(ctx, d_I, nx, ny, p, sigma_i, mode, out);
  size_t mark = ctx->arena.off;
  int nxx = nx / 2, nyy = ny / 2;
  float *d_Iz = ctx->arena.get<float>((size_t)nxx * nyy);
  B2F_ARENA_CHECK(ctx);
  int rc = harris_decimate2(ctx, d_I, d_Iz, nx, ny, ctx->stream);
  if (rc != B2F_OK) return rc;
  std::vector<Corner> cz;
  if ((rc = harris_scale(ctx, d_Iz, nxx, nyy, p, Nscales - 1, sigma_i / 2, mode, cz)) != B2F_OK) return rc;
  ctx->arena.off = mark;
  if ((rc = harris_one(ctx, d_I, nx, ny, p, sigma_i, mode, out)) != B2F_OK) return rc;
  std::vector<Corner> kept;                                         // select_corners, harris.cpp:443-465
  for (size_t i = 0; i < out.size(); i++) {
    size_t j = 0;
    for (; j < cz.size(); j++) {
      float dx = (cz[j].x - out[i].x / 2.);
      float dy = (cz[j].y - out[i].y / 2.);
      if (!(dx * dx + dy * dy > sigma_i * sigma_i)) break;
    }
    if (j < cz.size()) kept.push_back(out[i]);
  }
  out.swap(kept);
  return B2F_OK;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

void b2f_harris_default_params(b2f_harris_params *p) {   // rcpp_harris.cpp:19-32
  p->k = 0.06f; p->sigma_d = 1.0f; p->sigma_i = 2.5f; p->threshold = 130.f;
  p->gaussian = 1; p->gradient = 0; p->strategy = 0; p->Nselect = 1; p->measure = 0;
  p->Nscales = 1; p->precision = 1; p->cells = 10; p->verbose = 0; p->exact = 0;
}

// img_f (floats, as the reference narrows them) or img_d (R's doubles, narrowed on the device): exactly one is non-NULL
static int harris_host_any(b2f_ctx *ctx, const float *img_f, const double *img_d, int nx, int ny, const b2f_harris_params *p,
                           float **x, float **y, float **strength, int *n, const char *who) {
  if (!ctx || (!img_f && !img_d) || !p || !x || !y || !strength || !n) { set_error("%s: NULL argument", who); return B2F_EINVAL; }
  if (nx <= 0 || ny <= 0) { set_error("%s: bad size %dx%d", who, nx, ny); return B2F_EINVAL; }
  *x = *y = *strength = nullptr; *n = 0;
  B2F_CUDA(cudaSetDevice(ctx->device));
  size_t plane = (size_t)nx * ny;
  int cap = (nx / 2 + 1) * (ny / 2 + 1);
  // pyramid levels share the arena: bound by 2x the finest level
  int rc = arena_reserve(ctx, 2 * harris_scratch_bytes(1, nx, ny, p, cap) + align256(plane * 4) + (img_d ? align256(plane * 8) : 0));
  if (rc != B2F_OK) return rc;
  float *d_I = ctx->arena.get<float>(plane);
  B2F_ARENA_CHECK(ctx);
  if (img_f) B2F_CUDA(cudaMemcpyAsync(d_I, img_f, plane * sizeof(float), cudaMemcpyHostToDevice, ctx->stream));
  else {
    const size_t mark = ctx->arena.off;
    double *d_raw = ctx->arena.get<double>(plane);
    B2F_ARENA_CHECK(ctx);
    B2F_CUDA(cudaMemcpyAsync(d_raw, img_d, plane * sizeof(double), cudaMemcpyHostToDevice, ctx->stream));
    if ((rc = harris_double_to_float(ctx, d_raw, d_I, plane, ctx->stream)) != B2F_OK) return rc;
    ctx->arena.off = mark;                                          // (stream order keeps the staging plane alive until it is read)
  }
  std::vector<Corner> c;
  rc = harris_scale(ctx, d_I, nx, ny, p, p->Nscales, p->sigma_i, harris_mode(p), c);
  if (rc != B2F_OK) return rc;
  size_t m = c.size();
  float *ox = (float *)malloc(sizeof(float) * (m ? m : 1)), *oy = (float *)malloc(sizeof(float) * (m ? m : 1)),
        *os = (float *)malloc(sizeof(float) * (m ? m : 1));
  if (!ox || !oy || !os) { free(ox); free(oy); free(os); set_error("%s: out of host memory", who); return B2F_ENOMEM; }
  for (size_t i = 0; i < m; i++) { ox[i] = c[i].x; oy[i] = c[i].y; os[i] = c[i].R; }
  *x = ox; *y = oy; *strength = os; *n = (int)m;
  return B2F_OK;
}

int b2f_harris_host(b2f_ctx *ctx, const float *img, int nx, int ny, const b2f_harris_params *p,
                    float **x, float **y, float **strength, int *n) {
  return harris_host_any(ctx, img, nullptr, nx, ny, p, x, y, strength, n, "b2f_harris_host");
}

// detect_corners' NumericVector as it is (rcpp_harris.cpp:19-35): the doubles are uploaded and narrowed on the device
int b2f_harris_host_r64(b2f_ctx *ctx, const double *img, int nx, int ny, const b2f_harris_params *p,
                        float **x, float **y, float **strength, int *n) {
  return harris_host_any(ctx, nullptr, img, nx, ny, p, x, y, strength, n, "b2f_harris_host_r64");
}

int b2f_harris_response_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                            const b2f_harris_params *p, float *d_R, void *stream) {
  if (!ctx || !d_frames || !p || !d_R || n_frames <= 0 || nx <= 0 || ny <= 0) { set_error("b2f_harris_response_dev: bad argument"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  { int hrc = stream_handoff(ctx, stream, &st); if (hrc != B2F_OK) return hrc; }
  int exact = harris_mode(p) == MODE_STAGED ? 1 : 0;
  if (exact || !harris_fused_supported(nx, ny, p->sigma_d, p->sigma_i, p->gaussian)) {
    int rc = arena_reserve(ctx, harris_scratch_bytes(n_frames, nx, ny, p, 1));
    if (rc != B2F_OK) return rc;
  }
  return harris_response_device(ctx, d_frames, is_u8 != 0, n_frames, nx, ny, p, exact, d_R, st);
}

int b2f_harris_nms_dev(b2f_ctx *ctx, const float *d_R, int n_frames, int nx, int ny, float threshold, int radius,
                       int cap, int *d_xy, float *d_strength, int *d_counts, void *stream) {
  if (!ctx || !d_R || !d_xy || !d_strength || !d_counts || n_frames <= 0 || cap <= 0) { set_error("b2f_harris_nms_dev: bad argument"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  { int hrc = stream_handoff(ctx, stream, &st); if (hrc != B2F_OK) return hrc; }
  if (ny <= 2 * radius + 1 || nx <= 2 * radius + 1) {   // harris.cpp:151
    B2F_CUDA(cudaMemsetAsync(d_counts, 0, sizeof(int) * n_frames, st));
    return B2F_OK;
  }
  size_t need = align256((size_t)n_frames * ny * ceil_div(nx, 32) * 4) + align256((size_t)n_frames * ny * 4) +
                align256((size_t)n_frames * nx * ny) + 4096;
  int rc = arena_reserve(ctx, need);
  if (rc != B2F_OK) return rc;
  return harris_nms_device(ctx, d_R, n_frames, nx, ny, threshold, radius, cap, d_xy, d_strength, d_counts, st);
}

int b2f_harris_batch_u8(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int nx, int ny, const b2f_harris_params *p,
                        int cap, float *x, float *y, float *strength, int *counts) {
  if (!ctx || !frames || !p || !x || !y || !strength || !counts || n_frames <= 0 || nx <= 0 || ny <= 0 || cap <= 0) {
    set_error("b2f_harris_batch_u8: bad argument"); return B2F_EINVAL; }
  if (p->strategy != 0 || p->precision != 0 || p->Nscales > 1) {
    set_error("b2f_harris_batch_u8: the batch form emits all corners in raster order (strategy=0, precision=0, Nscales=1); "
              "use b2f_harris_host per frame for the other modes"); return B2F_EUNSUP; }
  return features_batch("b2f_harris_batch_u8", ctx, frames, 1, n_frames, ny, nx, p, cap, x, y, strength, counts,
                        nullptr, nullptr, nullptr, 0, 0, 0, nullptr);
}

int b2f_harris_corners_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                           const b2f_harris_params *p, int cap, int *d_xy, float *d_strength, int *d_counts, float *d_R,
                           void *stream) {
  if (!ctx || !d_frames || !p || !d_xy || !d_strength || !d_counts || n_frames <= 0 || nx <= 0 || ny <= 0 || cap <= 0) {
    set_error("b2f_harris_corners_dev: bad argument"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  { int hrc = stream_handoff(ctx, stream, &st); if (hrc != B2F_OK) return hrc; }
  int rc = arena_reserve(ctx, harris_scratch_bytes(n_frames, nx, ny, p, cap));
  if (rc != B2F_OK) return rc;
  return harris_corners_device(ctx, d_frames, is_u8 != 0, n_frames, nx, ny, p, cap, d_xy, d_strength, d_counts, d_R, st);
}

int b2f_harris_response_eps_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                                const b2f_harris_params *p, float *d_R, float *d_eps, void *stream) {
  if (!ctx || !d_frames || !p || !d_R || !d_eps || n_frames <= 0 || nx <= 0 || ny <= 0) { set_error("b2f_harris_response_eps_dev: bad argument"); return B2F_EINVAL; }
  if (!harris_fused_supported(nx, ny, p->sigma_d, p->sigma_i, p->gaussian)) { set_error("b2f_harris_response_eps_dev: no fused kernel for these parameters"); return B2F_EUNSUP; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  { int hrc = stream_handoff(ctx, stream, &st); if (hrc != B2F_OK) return hrc; }
  B2F_CUDA(cudaMemsetAsync(d_eps, 0, sizeof(float) * (size_t)n_frames * ((nx + 7) / 8) * ((ny + 7) / 8), st));
  return harris_fused_launch(ctx, d_frames, is_u8 != 0, n_frames, nx, ny, p, d_R, reinterpret_cast<unsigned *>(d_eps), false, st);
}

int b2f_harris_cert_stats(b2f_ctx *ctx, unsigned long long *out4) {
  if (!ctx || !out4) { set_error("b2f_harris_cert_stats: NULL argument"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  return harris_cert_stats(ctx, out4, ctx->stream);
}

}  // extern "C"
