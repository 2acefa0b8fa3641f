// nlmeans.cu — non-local means denoising of image.DenoiseNLMeans (rcpp_nlmeans -> nlmeans_ipol; the algorithm of
// Buades, Coll & Morel, IPOL 2011, doi:10.5201/ipol.2011.bcm_nlm), bit-identical to the reference run serially.
// Every float operation is an explicit round-to-nearest intrinsic: the reference is compiled without FMA contraction.
//   nlm_patch_kernel<WIN, C>  one thread per centre pixel of a band of centre rows.  The CTA stages the input region
//                             its 32x4 centres can reach (tile + bloc + win) in shared memory, then each thread walks
//                             its candidates j-outer / i-inner: patch distance (per channel, rows then columns,
//                             channel sums added in channel order), LUT weight, running maximum and total, and the
//                             weighted patch sums, all in the reference's visiting order.  It writes the normalised
//                             patch acc / total (or marks the centre invalid when total <= 1e-8f).  WIN >= 0 keeps
//                             the (2WIN+1)^2*C sums in registers; WIN = -1 (any other window) keeps them in the
//                             band buffer in global memory.
//   nlm_gather_kernel<C>      one thread per output pixel: adds the normalised patches of the centres of the band
//                             that cover it, in centre raster order, to the pixel's running sum and count.  Bands are
//                             processed in row order, so each pixel's sum runs through all its centres in raster
//                             order exactly as the reference's fpO[il] += ... does.
//   nlm_final_kernel<C>       out = sum / count, or the input pixel where no centre contributed.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <mutex>

namespace b2f {

constexpr int NL_TX = 32, NL_TY = 4;                    // centres per CTA of nlm_patch_kernel
constexpr int NL_LUT = 30000;                           // LUTMAX * LUTPRECISION entries of exp(-x)
constexpr size_t NL_BAND_BYTES = (size_t)256 << 20;     // normalised patches of one band of centre rows
constexpr int NL_SMEM_MAX = 160 * 1024;                 // staging larger than this reads the input from global memory
constexpr int NL_WIN_MAX = 10000;                       // keeps C*(2win+1)^2 inside an int, as the reference needs

struct NlmArgs {
  const float *in;            // [n][C][H][W]
  float *norm;                // [n][C][E][rows][W] normalised patches of the band's centres
  unsigned char *valid;       // [n][rows][W] 1 where total > fTiny
  const float *lut;           // NL_LUT floats
  int W, H, win, bloc;        // win = the largest patch radius any centre of the frame can have
  int y0, rows;               // the band: centre rows [y0, y0 + rows)
  float offset, fh2;          // 2*icwl*sigma^2 and (filter*sigma)^2*icwl, computed on the host like the reference
  int stage;                  // 1 = stage the reachable input region in shared memory
};

// wxSLUT (libauxiliar.cpp): the interpolation is done in double and rounded to float once.  A NaN distance (0 / 0 when
// filter*sigma is 0) indexes the reference's table out of bounds; here it weighs 0.
__device__ __forceinline__ float nl_slut(float d, const float *__restrict__ lut) {
  if (!(d < 29.0f)) return 0.0f;
  const double t = __dmul_rn((double)d, 1000.0);
  const int x = (int)floor(t);
  const float y1 = __ldg(lut + x), y2 = __ldg(lut + x + 1);
  return __double2float_rn(__dadd_rn((double)y1, __dmul_rn((double)__fsub_rn(y2, y1), __dsub_rn(t, (double)x))));
}

template <int WIN, int C>
__global__ void __launch_bounds__(NL_TX * NL_TY) nlm_patch_kernel(NlmArgs a) {
  extern __shared__ float sm[];
  const int win = WIN >= 0 ? WIN : a.win;
  const int side = 2 * win + 1, E = side * side;
  const int W = a.W, H = a.H, f = blockIdx.z;
  const int bx0 = blockIdx.x * NL_TX, by0 = a.y0 + blockIdx.y * NL_TY;
  const float *fin = a.in + (size_t)f * C * W * H;
  const float *src = fin;
  int ox = 0, oy = 0, pitch = W;
  size_t cs = (size_t)W * H;
  if (a.stage) {
    const int R = a.bloc + win;
    const int rx0 = max(0, bx0 - R), rx1 = min(W - 1, bx0 + NL_TX - 1 + R);
    const int ry0 = max(0, by0 - R), ry1 = min(H - 1, by0 + NL_TY - 1 + R);
    const int rw = rx1 - rx0 + 1, rn = rw * (ry1 - ry0 + 1);
    for (int c = 0; c < C; c++)
      for (int k = threadIdx.y * NL_TX + threadIdx.x; k < rn; k += NL_TX * NL_TY)
        sm[c * rn + k] = fin[(size_t)c * W * H + (size_t)(ry0 + k / rw) * W + rx0 + k % rw];
    __syncthreads();
    src = sm; ox = rx0; oy = ry0; pitch = rw; cs = rn;
  }
  const int x = bx0 + threadIdx.x, y = by0 + threadIdx.y;
  if (x >= W || y >= a.y0 + a.rows) return;

  const int w0 = min(min(a.win, min(W - 1 - x, H - 1 - y)), min(x, y));
  const int imin = max(x - a.bloc, w0), jmin = max(y - a.bloc, w0);
  const int imax = min(x + a.bloc, W - 1 - w0), jmax = min(y + a.bloc, H - 1 - w0);
  const int lim = WIN >= 0 ? WIN : w0;                  // loop bound: compile-time for the specialisations
  const size_t bplane = (size_t)a.rows * W;
  float *gslot = a.norm + (size_t)f * C * E * bplane + (size_t)(y - a.y0) * W + x;   // + (c*E + e) * bplane
  constexpr int NACC = WIN >= 0 ? C * (2 * WIN + 1) * (2 * WIN + 1) : 1;
  float racc[NACC];
#define NL_ACC(c, e) (WIN >= 0 ? racc[(c) * E + (e)] : gslot[((size_t)(c) * E + (e)) * bplane])
#define NL_IN(c, px, py) src[(size_t)(c) * cs + (size_t)((py) - oy) * pitch + ((px) - ox)]
#pragma unroll
  for (int c = 0; c < C; c++)
#pragma unroll
    for (int s = -lim; s <= lim; s++)
#pragma unroll
      for (int r = -lim; r <= lim; r++)
        if (WIN < 0 || (abs(s) <= w0 && abs(r) <= w0)) NL_ACC(c, (win + s) * side + win + r) = 0.0f;

  float fmax_w = 0.0f, ftot = 0.0f;
  for (int j = jmin; j <= jmax; j++)
    for (int i = imin; i <= imax; i++) {
      if (i == x && j == y) continue;
      float dif = 0.0f;                                 // fiL2FloatDist, channel by channel
#pragma unroll
      for (int c = 0; c < C; c++) {
        float dist = 0.0f;
#pragma unroll
        for (int s = -lim; s <= lim; s++)
#pragma unroll
          for (int r = -lim; r <= lim; r++)
            if (WIN < 0 || (abs(s) <= w0 && abs(r) <= w0)) {
              const float t = __fsub_rn(NL_IN(c, x + r, y + s), NL_IN(c, i + r, j + s));
              dist = __fadd_rn(dist, __fmul_rn(t, t));
            }
        dif = __fadd_rn(dif, dist);
      }
      dif = __fsub_rn(dif, a.offset);
      dif = dif < 0.0f ? 0.0f : dif;                    // MAX(fDif - ..., 0.0f)
      const float w = nl_slut(__fdiv_rn(dif, a.fh2), a.lut);
      if (w > fmax_w) fmax_w = w;
      ftot = __fadd_rn(ftot, w);
#pragma unroll
      for (int c = 0; c < C; c++)
#pragma unroll
        for (int s = -lim; s <= lim; s++)
#pragma unroll
          for (int r = -lim; r <= lim; r++)
            if (WIN < 0 || (abs(s) <= w0 && abs(r) <= w0)) {
              const int e = (win + s) * side + win + r;
              NL_ACC(c, e) = __fadd_rn(NL_ACC(c, e), __fmul_rn(w, NL_IN(c, i + r, j + s)));
            }
    }
#pragma unroll
  for (int c = 0; c < C; c++)                           // the centre's own patch, weighted by the largest weight
#pragma unroll
    for (int s = -lim; s <= lim; s++)
#pragma unroll
      for (int r = -lim; r <= lim; r++)
        if (WIN < 0 || (abs(s) <= w0 && abs(r) <= w0)) {
          const int e = (win + s) * side + win + r;
          NL_ACC(c, e) = __fadd_rn(NL_ACC(c, e), __fmul_rn(fmax_w, NL_IN(c, x + r, y + s)));
        }
  ftot = __fadd_rn(ftot, fmax_w);
  const bool ok = ftot > 1e-8f;                         // fTiny
  a.valid[(size_t)f * bplane + (size_t)(y - a.y0) * W + x] = ok;
  if (!ok) return;
#pragma unroll
  for (int c = 0; c < C; c++)
#pragma unroll
    for (int s = -lim; s <= lim; s++)
#pragma unroll
      for (int r = -lim; r <= lim; r++)
        if (WIN < 0 || (abs(s) <= w0 && abs(r) <= w0)) {
          const int e = (win + s) * side + win + r;
          gslot[((size_t)c * E + e) * bplane] = __fdiv_rn(NL_ACC(c, e), ftot);
        }
#undef NL_ACC
#undef NL_IN
}

// Pixel rows [py0, py0 + gridDim.y) receive the terms of the band's centres.
template <int C>
__global__ void __launch_bounds__(256) nlm_gather_kernel(const float *__restrict__ norm, const unsigned char *__restrict__ valid,
                                                         float *__restrict__ acc, int *__restrict__ cnt, int W, int H, int win,
                                                         int y0, int rows, int py0) {
  const int px = blockIdx.x * 256 + threadIdx.x, py = py0 + blockIdx.y, f = blockIdx.z;
  if (px >= W) return;
  const int side = 2 * win + 1, E = side * side;
  const size_t plane = (size_t)W * H, bplane = (size_t)rows * W;
  const float *fn = norm + (size_t)f * C * E * bplane;
  const unsigned char *fv = valid + (size_t)f * bplane;
  float s[C];
  const size_t p = (size_t)py * W + px;
#pragma unroll
  for (int c = 0; c < C; c++) s[c] = acc[((size_t)f * C + c) * plane + p];
  int n = cnt[(size_t)f * plane + p];
  const int cy1 = min(y0 + rows - 1, py + win), cx1 = min(W - 1, px + win);
  for (int cy = max(y0, py - win); cy <= cy1; cy++)
    for (int cx = max(0, px - win); cx <= cx1; cx++) {
      const int w0 = min(min(win, min(W - 1 - cx, H - 1 - cy)), min(cx, cy));
      const int dx = px - cx, dy = py - cy;
      if (abs(dx) > w0 || abs(dy) > w0) continue;
      const size_t q = (size_t)(cy - y0) * W + cx;
      if (!fv[q]) continue;
      const int e = (win + dy) * side + win + dx;
#pragma unroll
      for (int c = 0; c < C; c++) s[c] = __fadd_rn(s[c], fn[((size_t)c * E + e) * bplane + q]);
      n++;
    }
#pragma unroll
  for (int c = 0; c < C; c++) acc[((size_t)f * C + c) * plane + p] = s[c];
  cnt[(size_t)f * plane + p] = n;
}

template <int C>
__global__ void __launch_bounds__(256) nlm_final_kernel(const float *__restrict__ in, const float *__restrict__ acc,
                                                        const int *__restrict__ cnt, float *__restrict__ out, size_t plane) {
  const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x, f = blockIdx.y;
  if (p >= plane) return;
  const int n = cnt[f * plane + p];
#pragma unroll
  for (int c = 0; c < C; c++) {
    const size_t k = (f * C + c) * plane + p;
    out[k] = n > 0 ? __fdiv_rn(acc[k], (float)n) : in[k];
  }
}

// u8 [n][cin][H][W] or int32 (the same layout) -> float [n][C][H][W], the first C planes of each frame
template <typename T>
__global__ void nlm_widen_kernel(const T *__restrict__ src, float *__restrict__ dst, size_t plane, int cin, int C) {
  const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x, f = blockIdx.y / C, c = blockIdx.y % C;
  if (p >= plane) return;
  dst[(f * C + c) * plane + p] = (float)src[(f * cin + c) * plane + p];
}

// flag = 1 when the three planes differ somewhere (rcpp_denoisenlmeans.cpp's colour test)
__global__ void nlm_colour_kernel(const float *__restrict__ in, size_t plane, int *__restrict__ flag) {
  const size_t p = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (p >= plane) return;
  const float v = in[p];
  if (v != in[plane + p] || v != in[2 * plane + p]) *flag = 1;
}

// lut[i] = expf(-(float)i / 1000.0) with the host's libm, as wxFillExpLut computes it
static const std::vector<float> &nl_host_lut() {
  static std::vector<float> lut;
  static std::once_flag once;
  std::call_once(once, [] {
    lut.resize(NL_LUT);
    for (int i = 0; i < NL_LUT; i++) lut[i] = expf((float)(-(float)i / 1000.0));
  });
  return lut;
}

static int nl_ensure_lut(b2f_ctx *ctx, cudaStream_t st) {
  if (ctx->nlmeans_lut) return B2F_OK;
  void *p = nullptr;
  B2F_CUDA(cudaMalloc(&p, NL_LUT * sizeof(float)));
  const cudaError_t e = cudaMemcpyAsync(p, nl_host_lut().data(), NL_LUT * sizeof(float), cudaMemcpyHostToDevice, st);
  if (e != cudaSuccess) { cudaFree(p); set_error("nlmeans: LUT upload failed: %s", cudaGetErrorString(e)); return B2F_ECUDA; }
  ctx->nlmeans_lut = p;
  return B2F_OK;
}

static int nl_map_channels(int channels) { return channels == 2 ? 1 : channels > 3 ? 3 : channels; }

// Largest patch radius a centre of a W x H frame can have: w0 = min(win, x, y, W-1-x, H-1-y).
static int nl_eff_win(int win, int W, int H) { return std::min(win, (std::min(W, H) - 1) / 2); }

// Device scratch of one call, and the centre rows per band: n frames narrowed to cin float planes, C of them denoised
// (C = cin except after the colour test of the _host_r32 entry); host = 1 adds that entry's int32 upload, colour flag and
// float result.  The one bound that sizes the arena for every entry.
size_t nlmeans_scratch_bytes(int n, int cin, int C, int W, int H, int weff, int host, int *band_rows) {
  const size_t plane = (size_t)W * H, E = (size_t)(2 * weff + 1) * (2 * weff + 1);
  const size_t row = (size_t)n * W * (C * E * 4 + 1);
  const int rows = (int)std::max<size_t>(1, std::min<size_t>((size_t)H, NL_BAND_BYTES / row));
  if (band_rows) *band_rows = rows;
  size_t b = align256((size_t)n * cin * plane * 4)             // narrowed input
           + align256((size_t)n * C * plane * 4)               // running sums
           + align256((size_t)n * plane * 4)                   // counts
           + align256(C * E * 4 * (size_t)n * rows * W) + align256((size_t)n * rows * W);
  if (host) b += align256((size_t)n * cin * plane * 4) + 256 + align256((size_t)n * C * plane * 4);
  return b;
}

static int nl_check(const char *who, int n, int channels, int W, int H, int win, int bloc) {
  if (n <= 0 || W <= 0 || H <= 0) { set_error("%s: bad size %d x %dx%d", who, n, W, H); return B2F_EINVAL; }
  if (channels <= 0) { set_error("%s: channels must be positive (got %d)", who, channels); return B2F_EINVAL; }
  if ((long long)W * H * nl_map_channels(channels) > 2147483647LL) {
    set_error("%s: %dx%dx%d overflows the int indexing of the reference", who, W, H, channels);
    return B2F_EUNSUP;
  }
  if (win < 0 || bloc < 0) { set_error("%s: win and bloc must be >= 0 (got %d, %d)", who, win, bloc); return B2F_EINVAL; }
  if (win > NL_WIN_MAX) { set_error("%s: win %d > %d overflows the patch size of the reference", who, win, NL_WIN_MAX); return B2F_EUNSUP; }
  return B2F_OK;
}

template <int WIN, int C>
static void nl_launch_patch(const NlmArgs &a, dim3 grid, size_t smem, cudaStream_t st) {
  if (smem > 48 * 1024) cudaFuncSetAttribute(nlm_patch_kernel<WIN, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  nlm_patch_kernel<WIN, C><<<grid, dim3(NL_TX, NL_TY), smem, st>>>(a);
}

// d_in: n frames of C float planes (already narrowed) -> d_out the same layout.  The arena is reserved by the caller.
static int nlm_device(b2f_ctx *ctx, const float *d_in, int n, int C, int W, int H, int win, int bloc, float sigma,
                      float filter, float *d_out, cudaStream_t st) {
  const int weff = nl_eff_win(win, W, H), E = (2 * weff + 1) * (2 * weff + 1);
  bloc = std::min(bloc, std::max(W, H));                // a wider search window reaches no further pixel
  int rows = 1;
  nlmeans_scratch_bytes(n, C, C, W, H, weff, 0, &rows);
  const size_t plane = (size_t)W * H;
  float *acc = ctx->arena.get<float>((size_t)n * C * plane);
  int *cnt = ctx->arena.get<int>((size_t)n * plane);
  float *norm = ctx->arena.get<float>((size_t)C * E * n * rows * W);
  unsigned char *valid = ctx->arena.get<unsigned char>((size_t)n * rows * W);
  B2F_ARENA_CHECK(ctx);
  int rc = nl_ensure_lut(ctx, st);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaMemsetAsync(acc, 0, sizeof(float) * n * C * plane, st));
  B2F_CUDA(cudaMemsetAsync(cnt, 0, sizeof(int) * n * plane, st));

  // nlmeans_ipol's derived values, in its float operation order
  const int icwl = C * (2 * win + 1) * (2 * win + 1);
  const float fsigma2 = sigma * sigma;
  const float fh = filter * sigma;
  float fh2 = fh * fh;
  fh2 *= (float)icwl;
  const float offset = 2.0f * (float)icwl * fsigma2;

  const int R = bloc + weff;
  const size_t smem = (size_t)C * (NL_TX + 2 * R) * (NL_TY + 2 * R) * sizeof(float);
  const bool stage = smem <= (size_t)NL_SMEM_MAX;
  for (int y0 = 0; y0 < H; y0 += rows) {
    const int nr = std::min(rows, H - y0);
    NlmArgs a{d_in, norm, valid, (const float *)ctx->nlmeans_lut, W, H, weff, bloc, y0, nr, offset, fh2, stage ? 1 : 0};
    const dim3 grid(ceil_div(W, NL_TX), ceil_div(nr, NL_TY), n);
    const size_t sh = stage ? smem : 0;
    if (C == 1) {
      switch (weff) {
        case 1: nl_launch_patch<1, 1>(a, grid, sh, st); break;
        case 2: nl_launch_patch<2, 1>(a, grid, sh, st); break;
        case 3: nl_launch_patch<3, 1>(a, grid, sh, st); break;
        case 4: nl_launch_patch<4, 1>(a, grid, sh, st); break;
        case 5: nl_launch_patch<5, 1>(a, grid, sh, st); break;
        default: nl_launch_patch<-1, 1>(a, grid, sh, st);
      }
    } else {
      switch (weff) {
        case 1: nl_launch_patch<1, 3>(a, grid, sh, st); break;
        case 2: nl_launch_patch<2, 3>(a, grid, sh, st); break;
        case 3: nl_launch_patch<3, 3>(a, grid, sh, st); break;
        default: nl_launch_patch<-1, 3>(a, grid, sh, st);
      }
    }
    B2F_LAUNCH_CHECK(ctx);
    const int py0 = std::max(0, y0 - weff), py1 = std::min(H - 1, y0 + nr - 1 + weff);
    const dim3 gg(ceil_div(W, 256), py1 - py0 + 1, n);
    if (C == 1) nlm_gather_kernel<1><<<gg, 256, 0, st>>>(norm, valid, acc, cnt, W, H, weff, y0, nr, py0);
    else nlm_gather_kernel<3><<<gg, 256, 0, st>>>(norm, valid, acc, cnt, W, H, weff, y0, nr, py0);
    B2F_LAUNCH_CHECK(ctx);
  }
  const dim3 gf((unsigned)((plane + 255) / 256), n);
  if (C == 1) nlm_final_kernel<1><<<gf, 256, 0, st>>>(d_in, acc, cnt, d_out, plane);
  else nlm_final_kernel<3><<<gf, 256, 0, st>>>(d_in, acc, cnt, d_out, plane);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_nlmeans_resolve(int channels, float sigma, int args_auto, int *win, int *bloc, float *filter) {
  if (!win || !bloc || !filter) { set_error("b2f_nlmeans_resolve: bad argument"); return B2F_EINVAL; }
  if (channels <= 0) { set_error("b2f_nlmeans_resolve: channels must be positive (got %d)", channels); return B2F_EINVAL; }
  if (!args_auto) return B2F_OK;
  // rcpp_denoisenlmeans.cpp's table.  The first row of each table tests sigma > 0, so sigma <= 0 takes the last row.
  int w, b;
  float h;
  if (nl_map_channels(channels) == 1) {
    if (sigma > 0.0f && sigma <= 15.0f) { w = 1; b = 10; h = 0.4f; }
    else if (sigma > 15.0f && sigma <= 30.0f) { w = 2; b = 10; h = 0.4f; }
    else if (sigma > 30.0f && sigma <= 45.0f) { w = 3; b = 17; h = 0.35f; }
    else if (sigma > 45.0f && sigma <= 75.0f) { w = 4; b = 17; h = 0.35f; }
    else if (sigma <= 100.0f) { w = 5; b = 17; h = 0.30f; }
    else { set_error("error :: algorithm parametrized only for values of sigma less than 100.0"); return B2F_EINVAL; }
  } else {
    if (sigma > 0.0f && sigma <= 25.0f) { w = 1; b = 10; h = 0.55f; }
    else if (sigma > 25.0f && sigma <= 55.0f) { w = 2; b = 17; h = 0.4f; }
    else if (sigma <= 100.0f) { w = 3; b = 17; h = 0.35f; }
    else { set_error("error :: algorithm parametrized only for values of sigma less than 100.0"); return B2F_EINVAL; }
  }
  *win = w; *bloc = b; *filter = h;
  return B2F_OK;
}

int b2f_nlmeans_host_r32(b2f_ctx *ctx, const int32_t *image, int width, int height, int channels, float sigma, int args_auto,
                         int win, int bloc, float filter, float *out, int *out_channels, int *win_used, int *bloc_used,
                         float *filter_used) {
  if (!ctx || !image || !out || !out_channels || !win_used || !bloc_used || !filter_used) {
    set_error("b2f_nlmeans_host_r32: bad argument"); return B2F_EINVAL;
  }
  int rc = nl_check("b2f_nlmeans_host_r32", 1, channels, width, height, 0, 0);
  if (rc != B2F_OK) return rc;
  const int cin = nl_map_channels(channels);
  // The colour test may turn 3 planes into 1, which changes the table row; reserve for either outcome.
  size_t need = 0;
  for (int dc = 1; dc <= cin; dc += 2) {
    int w = win, b = bloc; float h = filter;
    if ((rc = b2f_nlmeans_resolve(dc, sigma, args_auto, &w, &b, &h)) != B2F_OK) return rc;
    if ((rc = nl_check("b2f_nlmeans_host_r32", 1, dc, width, height, w, b)) != B2F_OK) return rc;
    need = std::max(need, nlmeans_scratch_bytes(1, cin, dc, width, height, nl_eff_win(w, width, height), 1, nullptr));
  }
  B2F_CUDA(cudaSetDevice(ctx->device));
  if ((rc = arena_reserve(ctx, need)) != B2F_OK) return rc;
  const size_t plane = (size_t)width * height;
  int32_t *d_raw = ctx->arena.get<int32_t>((size_t)cin * plane);
  float *d_in = ctx->arena.get<float>((size_t)cin * plane);
  int *d_flag = ctx->arena.get<int>(1);
  B2F_ARENA_CHECK(ctx);
  cudaStream_t st = ctx->stream;
  B2F_CUDA(cudaMemcpyAsync(d_raw, image, (size_t)cin * plane * 4, cudaMemcpyHostToDevice, st));
  nlm_widen_kernel<int32_t><<<dim3((unsigned)((plane + 255) / 256), cin), 256, 0, st>>>(d_raw, d_in, plane, cin, cin);
  B2F_LAUNCH_CHECK(ctx);
  int dc = cin;
  if (cin == 3) {
    B2F_CUDA(cudaMemsetAsync(d_flag, 0, 4, st));
    nlm_colour_kernel<<<(unsigned)((plane + 255) / 256), 256, 0, st>>>(d_in, plane, d_flag);
    B2F_LAUNCH_CHECK(ctx);
    int colour = 0;
    B2F_CUDA(cudaMemcpyAsync(&colour, d_flag, 4, cudaMemcpyDeviceToHost, st));
    B2F_CUDA(cudaStreamSynchronize(st));
    if (!colour) dc = 1;
  }
  if ((rc = b2f_nlmeans_resolve(dc, sigma, args_auto, &win, &bloc, &filter)) != B2F_OK) return rc;
  float *d_out = ctx->arena.get<float>((size_t)dc * plane);
  B2F_ARENA_CHECK(ctx);
  if ((rc = nlm_device(ctx, d_in, 1, dc, width, height, win, bloc, sigma, filter, d_out, st)) != B2F_OK) return rc;
  B2F_CUDA(cudaMemcpyAsync(out, d_out, (size_t)dc * plane * 4, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  *out_channels = dc; *win_used = win; *bloc_used = bloc; *filter_used = filter;
  return B2F_OK;
}

int b2f_nlmeans_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int channels, int width, int height, int win, int bloc,
                    float sigma, float filter, float *d_out, void *stream) {
  if (!ctx || !d_frames || !d_out) { set_error("b2f_nlmeans_dev: bad argument"); return B2F_EINVAL; }
  int rc = nl_check("b2f_nlmeans_dev", n_frames, channels, width, height, win, bloc);
  if (rc != B2F_OK) return rc;
  const int dc = nl_map_channels(channels);
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  const int weff = nl_eff_win(win, width, height);
  if ((rc = arena_reserve(ctx, nlmeans_scratch_bytes(n_frames, channels, dc, width, height, weff, 0, nullptr))) != B2F_OK) return rc;
  const size_t plane = (size_t)width * height;
  float *d_in = ctx->arena.get<float>((size_t)n_frames * dc * plane);
  B2F_ARENA_CHECK(ctx);
  nlm_widen_kernel<uint8_t><<<dim3((unsigned)((plane + 255) / 256), n_frames * dc), 256, 0, st>>>(d_frames, d_in, plane, channels, dc);
  B2F_LAUNCH_CHECK(ctx);
  return nlm_device(ctx, d_in, n_frames, dc, width, height, win, bloc, sigma, filter, d_out, st);
}

}  // extern "C"
