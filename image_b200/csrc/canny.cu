// canny.cu — the Canny edge path (image.CannyEdges; SURVEY.md §8a rows C1-C5).
//
//   canny_blur_kernel      circular Gaussian blur, u8 -> float-rounded plane.  The reference runs a
//                          2-D FFT (tools.c:89-202); this is the same circular convolution evaluated
//                          directly: separable, double accumulation in a FIXED order (centre tap, then
//                          symmetric pairs by increasing distance), narrowed to float exactly like
//                          tools.c:129.  One CTA = 32x128 output tile, row pass into shared memory,
//                          column pass out of it; wrap-around addressing (tools.c:151-155).
//   canny_grad_nms_spec2_kernel
//                          gradient (rcpp_canny.cpp:153-175), then the interpolated non-maximum suppression
//                          of maxima()/bilin() (rcpp_canny.cpp:65-106) -> class 0/1/2 per pixel, speculated in
//                          fp32 and certified, undecided pixels redone in double with glibc's hypot
//                          reproduced operation by operation.  Output: two bit masks per 32-pixel tile row
//                          (edge = class != 0, strong = class 2).
//   hysteresis             union-find over the 8-neighbourhood of class!=0 pixels (the reference's
//                          adsf_* disjoint-set forest, adsf.c:17-50, rcpp_canny.cpp:184-215) on runs of
//                          the bit masks: tile-local in shared memory, then across tile seams on per-tile
//                          component ids with lock-free atomicMin links; a component survives iff it
//                          holds a class-2 pixel.
//   All arithmetic that feeds a comparison is IEEE double with explicit rounding intrinsics, i.e. no
//   FMA contraction, because the edge map has to come out bit-identical.
#include "common.cuh"
#include <cmath>
#include <vector>

namespace b2f {

constexpr int CANNY_MAXR = 64;       // taps beyond this radius use the generic (unrolled-less) path
struct CannyTaps {
  double w[CANNY_MAXR + 1];          // w[k] for distance k (symmetric list)
  int R;
};

// ------------------------------------------------------------------------------------------ blur
constexpr int CB_TW = 32, CB_TH = 64, CB_NT = 256;     // (64+2R) x (32+2R) doubles + row buffer = 65 KB at R=13: 3 CTAs / SM

__device__ __forceinline__ int wrap_index(int p, int n) {   // circular addressing, tools.c:151-155
  while (p < 0) p += n;
  while (p >= n) p -= n;
  return p;
}

// Shared memory: the input tile is converted to double ONCE at load time (u8 -> double is exact),
// so both passes are pure DADD/DMUL streams: pair sum, product, accumulate (40 fp64 ops / output).
template <int RT>
__global__ void __launch_bounds__(CB_NT, 3)
canny_blur_kernel(const unsigned char *__restrict__ frames, float *__restrict__ out, int nx, int ny,
                  const __grid_constant__ CannyTaps tx, const __grid_constant__ CannyTaps ty) {
  extern __shared__ __align__(16) double smem_d[];
  const int RX = RT ? RT : tx.R, RY = RT ? RT : ty.R;
  const int TILE_H = CB_TH + 2 * RY, TILE_W = CB_TW + 2 * RX;
  const int TP = (TILE_W + 1) & ~1;                       // pitch in doubles, even (16-byte rows)
  double *rowbuf = smem_d;                                // [TILE_H][CB_TW]
  double *tile = smem_d + (size_t)TILE_H * CB_TW;         // [TILE_H][TP]
  const int x0 = blockIdx.x * CB_TW, y0 = blockIdx.y * CB_TH;
  const unsigned char *src = frames + (size_t)blockIdx.z * nx * ny;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // ---- load with wrap-around: a warp streams whole tile rows
  //      (column offsets are per lane and hoisted; 6 rows are fetched per batch so that up to 18
  //       independent byte loads are in flight per thread instead of one load-use chain per row)
  {
    constexpr int MAXC = 3;                               // covers TILE_W <= 96 (RX <= 32); wider tiles loop
    int cofs[MAXC];
#pragma unroll
    for (int q = 0; q < MAXC; q++) cofs[q] = wrap_index(x0 - RX + lane + 32 * q, nx);
    constexpr int RBATCH = 6;
    for (int r0 = warp; r0 < TILE_H; r0 += (CB_NT / 32) * RBATCH) {
      unsigned char b[RBATCH][MAXC];
#pragma unroll
      for (int k = 0; k < RBATCH; k++) {
        const int r = r0 + (CB_NT / 32) * k;
        const unsigned char *row = src + (size_t)wrap_index(y0 - RY + min(r, TILE_H - 1), ny) * nx;
#pragma unroll
        for (int q = 0; q < MAXC; q++) b[k][q] = (lane + 32 * q < TILE_W) ? __ldg(row + cofs[q]) : (unsigned char)0;
      }
#pragma unroll
      for (int k = 0; k < RBATCH; k++) {
        const int r = r0 + (CB_NT / 32) * k;
        if (r < TILE_H) {
#pragma unroll
          for (int q = 0; q < MAXC; q++) if (lane + 32 * q < TILE_W) tile[r * TP + lane + 32 * q] = (double)b[k][q];
        }
      }
    }
    for (int r = warp; r < TILE_H; r += CB_NT / 32) {     // columns beyond 96 (very large s only)
      const unsigned char *row = src + (size_t)wrap_index(y0 - RY + r, ny) * nx;
      for (int c = lane + 32 * MAXC; c < TILE_W; c += 32) tile[r * TP + c] = (double)__ldg(row + wrap_index(x0 - RX + c, nx));
    }
  }
  __syncthreads();
  // ---- row pass: rowbuf[r][c] = w0*v0 + sum_k wk*(v[-k]+v[+k]); 4 outputs per thread when RT>0
  if (RT) {
    constexpr int RR = RT ? RT : 1;
    constexpr int NV = 4 + 2 * RR;                         // inputs of 4 consecutive outputs
    for (int it = threadIdx.x; it < TILE_H * (CB_TW / 4); it += CB_NT) {
      const int r = it / (CB_TW / 4), g = it - r * (CB_TW / 4);
      const double *p = tile + r * TP + 4 * g;             // output col j uses tile cols j .. j+2R
      double v[NV];
#pragma unroll
      for (int q = 0; q < NV / 2; q++) { double2 t = *reinterpret_cast<const double2 *>(p + 2 * q); v[2 * q] = t.x; v[2 * q + 1] = t.y; }
      double o[4];
#pragma unroll
      for (int j = 0; j < 4; j++) {
        double acc = __dmul_rn(tx.w[0], v[j + RR]);
#pragma unroll
        for (int k = 1; k <= RR; k++) acc = __fma_rn(tx.w[k], __dadd_rn(v[j + RR - k], v[j + RR + k]), acc);
        o[j] = acc;
      }
      double *d = rowbuf + r * CB_TW + 4 * g;
      *reinterpret_cast<double2 *>(d) = make_double2(o[0], o[1]);
      *reinterpret_cast<double2 *>(d + 2) = make_double2(o[2], o[3]);
    }
  } else {
    for (int r = warp; r < TILE_H; r += CB_NT / 32) {
      const double *p = tile + r * TP + lane + RX;
      double acc = __dmul_rn(tx.w[0], p[0]);
      for (int k = 1; k <= RX; k++) acc = __fma_rn(tx.w[k], __dadd_rn(p[-k], p[k]), acc);
      rowbuf[r * CB_TW + lane] = acc;
    }
  }
  __syncthreads();
  // ---- column pass, register-blocked 8 rows per thread, then narrow to float (tools.c:129)
  {
    const int c = lane;
    const int gx = x0 + c;
    float *dst = out + (size_t)blockIdx.z * nx * ny;
    if (RT) {
      constexpr int RB = 8;
      constexpr int RR = RT ? RT : 1;
      for (int rg = warp; rg < CB_TH / RB; rg += CB_NT / 32) {
        double v[RB + 2 * RR];
#pragma unroll
        for (int q = 0; q < RB + 2 * RR; q++) v[q] = rowbuf[(rg * RB + q) * CB_TW + c];
#pragma unroll
        for (int j = 0; j < RB; j++) {
          double acc = __dmul_rn(ty.w[0], v[j + RR]);
#pragma unroll
          for (int k = 1; k <= RR; k++) acc = __fma_rn(ty.w[k], __dadd_rn(v[j + RR - k], v[j + RR + k]), acc);
          int gy = y0 + rg * RB + j;
          if (gx < nx && gy < ny) dst[(size_t)gy * nx + gx] = __double2float_rn(acc);
        }
      }
    } else {
      for (int r = warp; r < CB_TH; r += CB_NT / 32) {
        const double *p = rowbuf + (r + RY) * CB_TW + c;
        double acc = __dmul_rn(ty.w[0], p[0]);
        for (int k = 1; k <= RY; k++) acc = __fma_rn(ty.w[k], __dadd_rn(p[-k * CB_TW], p[k * CB_TW]), acc);
        int gy = y0 + r;
        if (gx < nx && gy < ny) dst[(size_t)gy * nx + gx] = __double2float_rn(acc);
      }
    }
  }
}

// ---- two-kernel variant for the default radius (s = 2 -> R = 13) ------------------------------
// Row pass straight from global memory: a thread produces 4 consecutive outputs of one row from 9
// aligned 32-bit loads; symmetric pair sums are formed as exact integers and converted with the
// 2^52 trick, so the pass is 14 DADD(convert) + 14 DMUL + 13 DADD per output.  Column pass: a CTA
// stages a (128+2R) x 32 tile of the double row sums in shared memory (batched loads) and each thread
// produces 8 consecutive rows of one column.  Same operation order as the tiled kernel / the oracle.
__device__ __forceinline__ double u32_to_double(unsigned s) {   // exact: (2^52 + s) - 2^52
  return __dadd_rn(__hiloint2double(0x43300000, (int)s), -4503599627370496.0);
}

template <int RR>
__global__ void __launch_bounds__(256)
canny_blur_rows_kernel(const unsigned char *__restrict__ frames, double *__restrict__ rowsum, int nx, int ny,
                       const __grid_constant__ CannyTaps tx) {
  const int y = blockIdx.y;
  const int x4 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  if (x4 >= nx) return;
  const unsigned char *row = frames + ((size_t)blockIdx.z * ny + y) * nx;
  constexpr int LEAD = (RR + 3) & ~3;                            // 16: first loaded byte is x4 - LEAD
  constexpr int NW = (LEAD + 4 + RR + 3) / 4;                    // 9 words cover x4-16 .. x4+19
  unsigned char b[NW * 4];
  const bool fast = (nx & 3) == 0 && NW * 4 <= nx && (reinterpret_cast<uintptr_t>(frames) & 3) == 0;
  if (fast) {     // nx % 4 == 0: the circular wrap keeps word alignment, so row ends need no byte path
    const unsigned *w = reinterpret_cast<const unsigned *>(row);
    const int nw = nx >> 2, w0 = (x4 - LEAD) >> 2;              // (arithmetic shift: x4 - LEAD may be negative)
    unsigned v[NW];
#pragma unroll
    for (int q = 0; q < NW; q++) {
      int wi = w0 + q;
      wi += wi < 0 ? nw : 0;
      wi -= wi >= nw ? nw : 0;
      v[q] = __ldg(w + wi);
    }
#pragma unroll
    for (int q = 0; q < NW; q++) { b[4 * q] = v[q] & 0xff; b[4 * q + 1] = (v[q] >> 8) & 0xff; b[4 * q + 2] = (v[q] >> 16) & 0xff; b[4 * q + 3] = v[q] >> 24; }
  } else {
#pragma unroll
    for (int q = 0; q < NW * 4; q++) b[q] = __ldg(row + wrap_index(x4 - LEAD + q, nx));
  }
  double o[4];
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int c = LEAD + j;
    double acc = __dmul_rn(tx.w[0], u32_to_double(b[c]));
#pragma unroll
    for (int k = 1; k <= RR; k++) acc = __fma_rn(tx.w[k], u32_to_double((unsigned)b[c - k] + (unsigned)b[c + k]), acc);
    o[j] = acc;
  }
  double *d = rowsum + ((size_t)blockIdx.z * ny + y) * nx + x4;
  if (x4 + 3 < nx && (nx & 1) == 0) {
    *reinterpret_cast<double2 *>(d) = make_double2(o[0], o[1]);
    *reinterpret_cast<double2 *>(d + 2) = make_double2(o[2], o[3]);
  } else {
#pragma unroll
    for (int j = 0; j < 4; j++) if (x4 + j < nx) d[j] = o[j];
  }
}

constexpr int CC_TW = 32, CC_TH = 128;
template <int RR>
__global__ void __launch_bounds__(256)
canny_blur_cols_kernel(const double *__restrict__ rowsum, float *__restrict__ out, int nx, int ny,
                       const __grid_constant__ CannyTaps ty) {
  extern __shared__ __align__(16) double smem_d[];              // [CC_TH + 2RR][CC_TW]
  constexpr int TILE_H = CC_TH + 2 * RR;
  const int x0 = blockIdx.x * CC_TW, y0 = blockIdx.y * CC_TH;
  const double *src = rowsum + (size_t)blockIdx.z * nx * ny;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gx = x0 + lane;
  const int cx = min(gx, nx - 1);
  {
    constexpr int RBATCH = 10;                                   // 10 rows in flight per thread
    for (int r0 = warp; r0 < TILE_H; r0 += 8 * RBATCH) {
      double v[RBATCH];
#pragma unroll
      for (int k = 0; k < RBATCH; k++) {
        const int r = min(r0 + 8 * k, TILE_H - 1);
        v[k] = __ldg(src + (size_t)wrap_index(y0 - RR + r, ny) * nx + cx);
      }
#pragma unroll
      for (int k = 0; k < RBATCH; k++) { const int r = r0 + 8 * k; if (r < TILE_H) smem_d[r * CC_TW + lane] = v[k]; }
    }
  }
  __syncthreads();
  float *dst = out + (size_t)blockIdx.z * nx * ny;
  constexpr int RB = 8;
  for (int rg = warp; rg < CC_TH / RB; rg += 8) {
    double v[RB + 2 * RR];
#pragma unroll
    for (int q = 0; q < RB + 2 * RR; q++) v[q] = smem_d[(rg * RB + q) * CC_TW + lane];
#pragma unroll
    for (int j = 0; j < RB; j++) {
      double acc = __dmul_rn(ty.w[0], v[j + RR]);
#pragma unroll
      for (int k = 1; k <= RR; k++) acc = __fma_rn(ty.w[k], __dadd_rn(v[j + RR - k], v[j + RR + k]), acc);
      const int gy = y0 + rg * RB + j;
      if (gx < nx && gy < ny) dst[(size_t)gy * nx + gx] = __double2float_rn(acc);
    }
  }
}

// Un-tiled fallback (tiny images whose wrapped kernel is not symmetric, or radii too large for the
// tile): one thread per pixel.  sym != 0: centre tap then symmetric pairs (the order of the tiled
// kernel and of the oracle); sym == 0: taps in ascending coordinate order (the oracle's order then).
struct TapList { const int *coord; const double *weight; int n; int sym; };
__global__ void canny_blur_generic_rows(const unsigned char *__restrict__ frames, double *__restrict__ tmp, int nx, int ny,
                                        TapList t) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= nx) return;
  const unsigned char *src = frames + (size_t)blockIdx.z * nx * ny + (size_t)y * nx;
  double acc;
  if (t.sym) {
    const int R = t.n / 2;
    acc = __dmul_rn(t.weight[R], (double)src[x]);
    for (int k = 1; k <= R; k++)
      acc = __fma_rn(t.weight[R + k], __dadd_rn((double)src[wrap_index(x - k, nx)], (double)src[wrap_index(x + k, nx)]), acc);
  } else {
    acc = 0;
    for (int i = 0; i < t.n; i++) acc = __fma_rn(t.weight[i], (double)src[wrap_index(x - t.coord[i], nx)], acc);
  }
  tmp[(size_t)blockIdx.z * nx * ny + (size_t)y * nx + x] = acc;
}
__global__ void canny_blur_generic_cols(const double *__restrict__ tmp, float *__restrict__ out, int nx, int ny, TapList t) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= nx) return;
  const double *src = tmp + (size_t)blockIdx.z * nx * ny + x;
  double acc;
  if (t.sym) {
    const int R = t.n / 2;
    acc = __dmul_rn(t.weight[R], src[(size_t)y * nx]);
    for (int k = 1; k <= R; k++)
      acc = __fma_rn(t.weight[R + k], __dadd_rn(src[(size_t)wrap_index(y - k, ny) * nx], src[(size_t)wrap_index(y + k, ny) * nx]), acc);
  } else {
    acc = 0;
    for (int i = 0; i < t.n; i++) acc = __fma_rn(t.weight[i], src[(size_t)wrap_index(y - t.coord[i], ny) * nx], acc);
  }
  out[(size_t)blockIdx.z * nx * ny + (size_t)y * nx + x] = __double2float_rn(acc);
}

// ------------------------------------------------------------------------------------------ gradient + NMS
// glibc 2.39 hypot for finite, moderate arguments (sysdeps/ieee754/dbl-64/e_hypot.c, non-FMA kernel),
// reproduced operation by operation so that grad is bit-identical to the reference's libm call
// (rcpp_canny.cpp:172).  Verified against libm on 5e6 random inputs (DESIGN.md §5).
__device__ __forceinline__ double hypot_glibc(double x, double y) {
  x = fabs(x); y = fabs(y);
  double ax = x < y ? y : x, ay = x < y ? x : y;
  if (ax >= __dmul_rn(ay, 0x1p54)) return __dadd_rn(ax, ay);   // ay/EPS, exact power-of-two scaling
  double h = __dsqrt_rn(__dadd_rn(__dmul_rn(ax, ax), __dmul_rn(ay, ay)));
  double t1, t2;
  if (h <= __dmul_rn(2.0, ay)) {
    double delta = __dsub_rn(h, ay);
    t1 = __dmul_rn(ax, __dsub_rn(__dmul_rn(2.0, delta), ax));
    t2 = __dmul_rn(__dsub_rn(delta, __dmul_rn(2.0, __dsub_rn(ax, ay))), delta);
  } else {
    double delta = __dsub_rn(h, ax);
    t1 = __dmul_rn(__dmul_rn(2.0, delta), __dsub_rn(ax, __dmul_rn(2.0, ay)));
    t2 = __dadd_rn(__dmul_rn(__dsub_rn(__dmul_rn(4.0, delta), ay), ay), __dmul_rn(delta, delta));
  }
  return __dsub_rn(h, __ddiv_rn(__dadd_rn(t1, t2), __dmul_rn(2.0, h)));
}

constexpr int CG_T = 32, CG_NT = 256;

// ------------------------------------------------------------------------------------------ gradient + NMS
// The gradient (rcpp_canny.cpp:153-175) and the interpolated non-maximum suppression of maxima()/bilin()
// (rcpp_canny.cpp:65-106), one 32x32 tile per CTA, reached in two tiers:
//   tier 1 (every pixel, fp32): gradient, magnitude, direction and the two bilinear neighbours in
//           single precision, together with a bound on how far those values can be from the
//           reference's doubles.  If every comparison of rcpp_canny.cpp:97-103 (now vs prev / next /
//           low / high) is decided with a margin larger than the bound, the class is final.
//   tier 2 (the rare undecided pixel): the exact double evaluation of that pixel alone, including
//           glibc-exact hypot of its up to nine neighbour magnitudes.
// The classes are therefore those of the all-double oracle (tests/test_canny_certify_cpu.py checks the
// tier-1 bound against it).  Error budget of tier 1 (the float data are exact inputs): E is a per-tile
// bound on |d grad|; a bilinear value inherits it plus (|d cos| + |d sin|) * (spread of its four corner
// magnitudes) with |d cos|,|d sin| <= 2E/now + 2^-21.  The margins below are >= twice that.
//   * data tile 36x36 (clamped coordinates at load, so the gradient needs no clamping at all), gradient
//     tile 34x34;
//   * gradient: one thread per (column, strip of 5 rows) slides down its strip with the three columns of
//     the two previous rows in registers: 3 shared loads per pixel, row differences reused;
//   * direction: xt, yt lie in [-1, 1], so floor() is a sign test; the opposite neighbour mirrors the
//     cell and swaps the bilinear weights; approximate reciprocal / square root, their error is part of
//     the bound (4e-7*g; 5e-7 on the cosines).
// Output: the tile's classes as two bit masks per row, stored tile-major (see "hysteresis" below).
constexpr int SG_DW = CG_T + 4;   // data tile columns, origin (x0-2, y0-2)
constexpr int SG_DH = CG_T + 5;   // data tile rows (one more than needed: the 7 gradient strips are all 5 rows tall)
constexpr int SG_GW = CG_T + 2;   // gradient tile columns, origin (x0-1, y0-1)
constexpr int SG_GH = CG_T + 3;   // gradient tile rows (34 used + 1 never read)
constexpr int SG_K = 5;           // rows per gradient strip: 7 strips x 34 columns = 238 work items
__device__ __forceinline__ float rcp_approx(float x) { float r; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }
__device__ __forceinline__ float sqrt_approx(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

__device__ __forceinline__ void exact_hv2(const float *d, int accGrad, double &h, double &v) {   // pitch SG_DW
#define DD(dx, dy) ((double)d[(dy) * SG_DW + (dx)])
  if (accGrad) {
    h = __dmul_rn(2.0, __dsub_rn(DD(1, 0), DD(-1, 0)));
    h = __dadd_rn(h, DD(1, 1)); h = __dsub_rn(h, DD(-1, 1)); h = __dadd_rn(h, DD(1, -1)); h = __dsub_rn(h, DD(-1, -1));
    v = __dmul_rn(2.0, __dsub_rn(DD(0, 1), DD(0, -1)));
    v = __dadd_rn(v, DD(1, 1)); v = __dsub_rn(v, DD(1, -1)); v = __dadd_rn(v, DD(-1, 1)); v = __dsub_rn(v, DD(-1, -1));
  } else {
    h = __dsub_rn(DD(1, 0), DD(-1, 0));
    v = __dsub_rn(DD(0, 1), DD(0, -1));
  }
#undef DD
}

template <bool ACC>
__global__ void __launch_bounds__(CG_NT)
canny_grad_nms_spec2_kernel(const float *__restrict__ data, unsigned *__restrict__ emask, unsigned *__restrict__ smask, int nx, int ny,
                            int low_thr, int high_thr, unsigned long long *__restrict__ fallback_count) {
  __shared__ __align__(16) float sd[SG_DH * SG_DW];
  __shared__ float fg[SG_GH * SG_GW];
  __shared__ float2 fhv[SG_GH * SG_GW];
  __shared__ float s_emax[CG_NT / 32];
  __shared__ __align__(4) unsigned char scls[CG_T * CG_T];
  __shared__ unsigned short squeue[CG_T * CG_T];
  __shared__ double sg2[28 * 9];
  __shared__ int qn;
  const int x0 = blockIdx.x * CG_T, y0 = blockIdx.y * CG_T;
  const float *src = data + (size_t)blockIdx.z * nx * ny;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) qn = 0;
  if (x0 >= 2 && y0 >= 2 && x0 + SG_DW - 2 <= nx && y0 + SG_DH - 2 <= ny && (nx & 1) == 0) {
    // data tile inside the image: 18 float2 per row, three per thread, all loads before the stores
    const float *org = src + (size_t)(y0 - 2) * nx + (x0 - 2);
    float2 v[3];
    int so[3];
#pragma unroll
    for (int k = 0; k < 3; k++) {
      const int u = threadIdx.x + k * CG_NT;
      const int row = u / (SG_DW / 2), cu = u - row * (SG_DW / 2);
      so[k] = row * SG_DW + 2 * cu;
      v[k] = u < SG_DH * (SG_DW / 2) ? __ldg(reinterpret_cast<const float2 *>(org + (size_t)row * nx + 2 * cu)) : make_float2(0.f, 0.f);
    }
#pragma unroll
    for (int k = 0; k < 3; k++)
      if (threadIdx.x + k * CG_NT < SG_DH * (SG_DW / 2)) *reinterpret_cast<float2 *>(sd + so[k]) = v[k];
  } else {   // clamped coordinates
    const int c0 = min(max(x0 - 2 + lane, 0), nx - 1), c1 = min(max(x0 - 2 + lane + 32, 0), nx - 1);
    float a[5], b[5];
#pragma unroll
    for (int k = 0; k < 5; k++) {
      const int j = min(warp + 8 * k, SG_DH - 1);
      const float *row = src + (size_t)min(max(y0 - 2 + j, 0), ny - 1) * nx;
      a[k] = __ldg(row + c0);
      b[k] = lane < SG_DW - 32 ? __ldg(row + c1) : 0.f;
    }
#pragma unroll
    for (int k = 0; k < 5; k++) {
      const int j = warp + 8 * k;
      if (j < SG_DH) { sd[j * SG_DW + lane] = a[k]; if (lane < SG_DW - 32) sd[j * SG_DW + lane + 32] = b[k]; }
    }
  }
  __syncthreads();
  // ---- tier-1 gradient tile.  Differences first (exact or nearly so): the rounding error then scales with
  // the local contrast S = sum |terms|:  |dh|,|dv| <= 3*2^-24*S,  |d grad| <= sqrt2*max(|dh|,|dv|) + 1.8e-7*grad
  // (h*h+v*v and the approximate root).  E is about twice that; its tile maximum is this CTA's tolerance unit.
  float emax = 0.f;
  if (threadIdx.x < 7 * SG_GW) {
    const int strip = threadIdx.x / SG_GW, c = threadIdx.x - strip * SG_GW;
    const float *d = sd + strip * SG_K * SG_DW + c;   // data (row, col) = gradient pixel (row, col) shifted by (-1, -1)
    float l0 = d[0], m0 = d[1], q0 = d[2];
    float l1 = d[SG_DW], m1 = d[SG_DW + 1], q1 = d[SG_DW + 2];
    float dh0 = q0 - l0, dh1 = q1 - l1;
    int gi = strip * SG_K * SG_GW + c;
#pragma unroll
    for (int k = 0; k < SG_K; k++) {
      const float l2 = d[(k + 2) * SG_DW], m2 = d[(k + 2) * SG_DW + 1], q2 = d[(k + 2) * SG_DW + 2];
      const float dh2 = q2 - l2;
      float h, v, S;
      const float vy = m2 - m0;
      if (ACC) {
        const float vp = q2 - q0, vm = l2 - l0;
        h = fmaf(2.f, dh1, dh2 + dh0);
        v = fmaf(2.f, vy, vp + vm);
        S = fmaf(2.f, fabsf(dh1) + fabsf(vy), (fabsf(dh2) + fabsf(dh0)) + (fabsf(vp) + fabsf(vm)));
      } else {
        h = dh1; v = vy;
        S = fabsf(h) + fabsf(v);
      }
      const float g = sqrt_approx(fmaf(h, h, v * v));
      fg[gi + k * SG_GW] = g;
      fhv[gi + k * SG_GW] = make_float2(h, v);
      if (strip * SG_K + k < SG_GW) emax = fmaxf(emax, fmaf(6e-7f, S, 4e-7f * g));   // (row 34 is never read)
      l0 = l1; m0 = m1; q0 = q1; dh0 = dh1;
      l1 = l2; m1 = m2; q1 = q2; dh1 = dh2;
    }
  }
  for (int o = 16; o; o >>= 1) emax = fmaxf(emax, __shfl_xor_sync(0xffffffffu, emax, o));
  if (lane == 0) s_emax[warp] = emax;
  __syncthreads();
  float E = s_emax[0];
#pragma unroll
  for (int w = 1; w < CG_NT / 32; w++) E = fmaxf(E, s_emax[w]);
  E = fmaxf(E, 1e-7f);
  const bool interior = x0 >= 1 && y0 >= 1 && x0 + CG_T + 1 <= nx && y0 + CG_T + 1 <= ny;
  const float lowf = (float)low_thr, highf = (float)high_thr;
  const float T0 = 2.f * E;                                      // 2 x bound on |d grad| anywhere in this tile
#pragma unroll
  for (int k = 0; k < CG_T * CG_T / CG_NT; k++) {
    const int t = threadIdx.x + k * CG_NT;
    const int ly = t >> 5, lx = t & 31;
    const int gx = x0 + lx, gy = y0 + ly;
    unsigned char c = 0;
    const int ci = (ly + 1) * SG_GW + lx + 1;
    const float now = fg[ci];
    if (gx < nx && gy < ny && now >= lowf - T0) {                // below: certainly now <= low, class 0
      const float inv = rcp_approx(now);
      const float2 hv = fhv[ci];
      const float cs = hv.x * inv, sn = hv.y * inv;
      const float dcs = 8.f * fmaf(E, inv, 5e-7f);               // bound on |d cos|, |d sin| (x4 margin)
      // "+" neighbour at (cs, sn): cell corner and weights; the "-" neighbour mirrors the cell and swaps the weights
      const int ngx = cs < 0.f, ngy = sn < 0.f;
      const float wbx = cs + (float)ngx, wax = 1.f - wbx, wby = sn + (float)ngy, way = 1.f - wby;
      float p11, p12, p21, p22, m11, m12, m21, m22;
      if (interior) {
        const float *gp = fg + ci - ngy * SG_GW - ngx;
        const float *gm = fg + ci + (ngy - 1) * SG_GW + (ngx - 1);
        p11 = gp[0]; p12 = gp[1]; p21 = gp[SG_GW]; p22 = gp[SG_GW + 1];
        m11 = gm[0]; m12 = gm[1]; m21 = gm[SG_GW]; m22 = gm[SG_GW + 1];
      } else {     // value(): neighbour coordinates clamp to the image
        const int ox = x0 - 1, oy = y0 - 1;
        const int px1 = min(max(gx - ngx, 0), nx - 1) - ox, px2 = min(max(gx - ngx + 1, 0), nx - 1) - ox;
        const int py1 = min(max(gy - ngy, 0), ny - 1) - oy, py2 = min(max(gy - ngy + 1, 0), ny - 1) - oy;
        const int mx1 = min(max(gx + ngx - 1, 0), nx - 1) - ox, mx2 = min(max(gx + ngx, 0), nx - 1) - ox;
        const int my1 = min(max(gy + ngy - 1, 0), ny - 1) - oy, my2 = min(max(gy + ngy, 0), ny - 1) - oy;
        p11 = fg[py1 * SG_GW + px1]; p12 = fg[py1 * SG_GW + px2]; p21 = fg[py2 * SG_GW + px1]; p22 = fg[py2 * SG_GW + px2];
        m11 = fg[my1 * SG_GW + mx1]; m12 = fg[my1 * SG_GW + mx2]; m21 = fg[my2 * SG_GW + mx1]; m22 = fg[my2 * SG_GW + mx2];
      }
      const float nbp = way * fmaf(wax, p11, wbx * p12) + wby * fmaf(wax, p21, wbx * p22);
      const float nbm = wby * fmaf(wbx, m11, wax * m12) + way * fmaf(wbx, m21, wax * m22);
      const float spp = fmaxf(fmaxf(p11, p12), fmaxf(p21, p22)) - fminf(fminf(p11, p12), fminf(p21, p22));
      const float spm = fmaxf(fmaxf(m11, m12), fmaxf(m21, m22)) - fminf(fminf(m11, m12), fminf(m21, m22));
      const float tolp = fmaf(dcs, spp, 2.f * T0), tolm = fmaf(dcs, spm, 2.f * T0);
      // undecided: now within the bound of `low`; a cosine within its error of 0 (the reference's floor() is
      // ambiguous there); a comparison with a neighbour or with `high` inside the bound
      const bool amb = now <= lowf + T0 || fminf(fabsf(cs), fabsf(sn)) <= dcs;
      const bool sup = now < fmaxf(nbp - tolp, nbm - tolm);      // certainly suppressed
      const bool top = now > fmaxf(nbp + tolp, nbm + tolm);      // certainly a maximum
      const bool hi2 = now >= highf + T0, hi1 = now < highf - T0;
      const bool undecided = amb || (!sup && (!top || (!hi2 && !hi1)));
      c = (!undecided && !sup) ? (hi2 ? 2 : 1) : 0;
      if (undecided) squeue[atomicAdd(&qn, 1)] = (unsigned short)t;
    }
    scls[t] = c;
  }
  __syncthreads();
  // ---- tier 2: the undecided pixels of this tile.  Their exact magnitudes are needed on the 3x3 block around
  // each of them (the bilinear corners lie there): one thread per (pixel, block position) does one glibc-exact
  // hypot, then one thread per pixel finishes the reference's double arithmetic.
  const int nq = qn;
  double *eg = sg2;                                              // [chunk][9]
  for (int qb = 0; qb < nq; qb += 28) {
    const int nc = min(28, nq - qb);
    for (int i = threadIdx.x; i < nc * 9; i += CG_NT) {
      const int qi = i / 9, k = i - qi * 9;
      const int t = squeue[qb + qi], ly = t >> 5, lx = t & 31;
      const int px = min(max(x0 + lx + (k % 3) - 1, 0), nx - 1), py = min(max(y0 + ly + (k / 3) - 1, 0), ny - 1);
      double h, v;
      exact_hv2(sd + (py - (y0 - 2)) * SG_DW + (px - (x0 - 2)), ACC, h, v);
      eg[i] = hypot_glibc(h, v);
    }
    __syncthreads();
    for (int qi = threadIdx.x; qi < nc; qi += CG_NT) {
      const int t = squeue[qb + qi], ly = t >> 5, lx = t & 31;
      const int gx = x0 + lx, gy = y0 + ly;
      const double *g9 = eg + qi * 9;
      double h, v;
      exact_hv2(sd + (gy - (y0 - 2)) * SG_DW + (gx - (x0 - 2)), ACC, h, v);
      const double now = g9[4];
      unsigned char c;
      if (now <= (double)low_thr) c = 0;
      else {
        double sn, cs;
        if (h == 0.0 || v == 0.0) { const double th = atan2(v, h); sincos(th, &sn, &cs); }
        else { const double inv = __ddiv_rn(1.0, now); cs = __dmul_rn(h, inv); sn = __dmul_rn(v, inv); }
        double nb[2];
        for (int s2 = 0; s2 < 2; s2++) {
          const double dir = s2 ? 1.0 : -1.0;
          const double xt = __dmul_rn(dir, cs), yt = __dmul_rn(dir, sn);
          const double x1 = floor(xt), x2 = __dadd_rn(x1, 1.0), y1 = floor(yt), y2 = __dadd_rn(y1, 1.0);
          auto G = [&](double ox, double oy) -> double {
            const int ix = (int)ox, iy = (int)oy;
            if (ix > 1 || iy > 1) return 0.0;                    // multiplied by a zero weight (xt or yt == 1)
            const int cxp = min(max(gx + ix, 0), nx - 1) - gx, cyp = min(max(gy + iy, 0), ny - 1) - gy;
            return g9[(cyp + 1) * 3 + (cxp + 1)];
          };
          const double wa = __dsub_rn(x2, xt), wb = __dsub_rn(xt, x1);
          const double g1 = __dadd_rn(__dmul_rn(wa, G(x1, y1)), __dmul_rn(wb, G(x2, y1)));
          const double g2 = __dadd_rn(__dmul_rn(wa, G(x1, y2)), __dmul_rn(wb, G(x2, y2)));
          nb[s2] = __dadd_rn(__dmul_rn(__dsub_rn(y2, yt), g1), __dmul_rn(__dsub_rn(yt, y1), g2));
        }
        if (now <= nb[0] || now <= nb[1]) c = 0;
        else c = now >= (double)high_thr ? 2 : 1;
      }
      scls[t] = c;
    }
    __syncthreads();
  }
  // ---- two ballots per tile row: edge = class != 0, strong = class == 2 (pixels outside the image are class 0)
  {
    const size_t t = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
#pragma unroll
    for (int k = 0; k < CG_T / (CG_NT / 32); k++) {
      const int ly = warp + (CG_NT / 32) * k;
      const unsigned char c = scls[ly * CG_T + lane];
      const unsigned e = __ballot_sync(0xffffffffu, c != 0), s = __ballot_sync(0xffffffffu, c == 2);
      if (lane == 0) { emask[CG_T * t + ly] = e; smask[CG_T * t + ly] = s; }
    }
  }
  if (fallback_count && threadIdx.x == 0 && nq) atomicAdd(fallback_count, (unsigned long long)nq);
}

// ------------------------------------------------------------------------------------------ hysteresis
// Union-find over the 8-neighbourhood of the class!=0 pixels (the reference's adsf_* disjoint-set forest,
// adsf.c:17-50, rcpp_canny.cpp:184-215); a component survives iff it holds a class-2 pixel.  Labels belong to
// horizontal RUNS of edge pixels, never to single pixels.  The hysteresis tiles are the 32x32 NMS tiles,
// tile t = (f*TY + ty)*TX + tx, and the passes exchange:
//   E[32t + r], S[32t + r]   row r of tile t as bit masks (bit x = column x): edge = class != 0, strong = class 2;
//                            bits past nx and rows past ny are 0 (canny_grad_nms_spec2_kernel)
//   ncomp[t]                 the number of 8-connected components of the tile's edge pixels (<= HYST_MAX_ROOTS)
//   runc[t][r][j]            the tile component of the j-th run (lowest first) of row r
//   parent, strong, keep     per component id 256t + c: the global forest (lock-free atomicMin links; a root is
//                            the smallest id of its set, as in adsf.c:31-40), "holds a class-2 pixel", and
//                            "its global component holds a class-2 pixel"
// Passes: hyst_local (tile components), hyst_seam (unions across tile borders), hyst_mark / hyst_resolve (a
// strong component marks its root; every component reads its root's mark), hyst_emit (edge map and counts).
__device__ __forceinline__ int uf_find(volatile int *L, int a) {
  int p = L[a];
  while (p != a) {
    int g = L[p];
    if (g != p) L[a] = g;          // path halving: parents only ever move to an ancestor
    a = p; p = g;
  }
  return a;
}
__device__ __forceinline__ int uf_find_ro(const volatile int *L, int a) {   // no path compression: safe beside plain stores
  int p = L[a];
  while (p != a) { a = p; p = L[a]; }
  return a;
}
__device__ __forceinline__ void uf_union(int *L, int a, int b) {
  while (true) {
    a = uf_find(L, a); b = uf_find(L, b);
    if (a == b) return;
    if (a < b) { int t = a; a = b; b = t; }     // a > b : link a under b
    int old = atomicMin(&L[a], b);
    if (old == a) return;
    a = old;                                     // a was linked elsewhere meanwhile: merge that set too
  }
}

constexpr int HT = CG_T;                              // hysteresis tile edge = NMS tile edge (one warp lane per row)
constexpr int HYST_MAX_RUNS = HT / 2;                 // runs in a 32-bit row
constexpr int HYST_MAX_ROOTS = (HT / 2) * (HT / 2);   // 8-connected components are >= 2 apart: isolated pixels on a 2-pixel lattice

__device__ __forceinline__ int run_start(unsigned bits, int x) {
  // first column of the run of set bits that contains bit x (bit x must be set)
  return x - __clz(~(bits << (31 - x))) + 1;
}
__device__ __forceinline__ int run_ordinal(unsigned bits, int x) {
  // ordinal, lowest first, of the run of set bits that contains bit x (bit x must be set): run heads at or below x, less one
  return __popc(bits & ~(bits << 1) & (0xffffffffu >> (31 - x))) - 1;
}
__device__ __forceinline__ unsigned run_mask_from(unsigned bits, int s) {   // the run of set bits of `bits` that starts at bit s
  const unsigned t = ~(bits >> s);                                         // first zero above s ...
  const int len = t ? __ffs(t) - 1 : 32;                                   // (bits >> s) shifts zeros in, so t != 0 unless s == 0 && bits == ~0
  return (len >= 32 ? 0xffffffffu : ((1u << len) - 1u)) << s;
}

// Tile components.  ONE WARP per tile (8 tiles per CTA), lane r on row r, working on runs:
//   * label slot r*16 + j is the j-th run of row r (peeled lowest first); a lane initialises its own slots;
//   * each run is linked (lock-free union, atomicMin on shared memory) to every run of the row above that
//     touches it 8-connectedly -- all 32 rows concurrently;
//   * the roots are numbered 0..n-1 in raster order of their heads (a warp scan: the numbering is deterministic);
//   * per run the component number goes to runc; per component the parent (itself) and the strong flag.
__global__ void __launch_bounds__(256)
hyst_local_kernel(const unsigned *__restrict__ E, const unsigned *__restrict__ S, unsigned char *__restrict__ runc,
                  int *__restrict__ ncomp, int *__restrict__ parent, unsigned char *__restrict__ strong, int n_tiles) {
  __shared__ int lab_all[8][HT * HYST_MAX_RUNS];
  __shared__ unsigned char num_all[8][HT * HYST_MAX_RUNS];     // root slot -> component number
  __shared__ __align__(8) unsigned char cst_all[8][HYST_MAX_ROOTS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int tile = blockIdx.x * 8 + warp;
  if (tile >= n_tiles) return;
  int *lab = lab_all[warp];
  unsigned char *num = num_all[warp], *cst = cst_all[warp];
  const unsigned emask = E[(size_t)HT * tile + lane], smask = S[(size_t)HT * tile + lane];
  if (!__any_sync(0xffffffffu, emask != 0)) { if (lane == 0) ncomp[tile] = 0; return; }   // empty tile
  const int nr = __popc(emask & ~(emask << 1)), s0 = lane * HYST_MAX_RUNS;
  for (int j = 0; j < nr; j++) lab[s0 + j] = s0 + j;
  reinterpret_cast<uint2 *>(cst)[lane] = make_uint2(0, 0);
  const unsigned up = __shfl_up_sync(0xffffffffu, emask, 1);
  __syncwarp();
  // ---- link every run to the touching runs of the row above.  Runs are peeled lowest first:
  //      low = lowest set bit, x = rem + low carries through the run, run = rem & ~x, rest = rem & x.
  if (lane > 0 && up) {
    int j = 0;
    for (unsigned rem = emask; rem; j++) {
      const unsigned low = rem & (0u - rem), x = rem + low, rm = rem & ~x;
      rem &= x;
      unsigned touch = up & (rm | (rm << 1) | (rm >> 1));
      while (touch) {
        const int us = run_start(up, __ffs(touch) - 1);
        const unsigned uhi = up >> us << us, ulow = 1u << us;                   // the up-run that starts at us
        touch &= ~(uhi & ~(uhi + ulow));
        uf_union(lab, s0 + j, s0 - HYST_MAX_RUNS + run_ordinal(up, us));
      }
    }
  }
  __syncwarp();
  // ---- flatten, and number the roots (the forest is final here: a run is a root iff its find returns itself)
  unsigned isroot = 0;
  for (int j = 0; j < nr; j++) {
    const int rt = uf_find(lab, s0 + j);
    lab[s0 + j] = rt;
    isroot |= (unsigned)(rt == s0 + j) << j;
  }
  const int mine = __popc(isroot);
  int incl = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  const int total = __shfl_sync(0xffffffffu, incl, 31);
  for (unsigned m = isroot; m; m &= m - 1) {
    const int j = __ffs(m) - 1;
    num[s0 + j] = (unsigned char)(incl - mine + __popc(isroot & ((1u << j) - 1u)));
  }
  __syncwarp();
  // ---- per run: its component number (packed 8 per 64-bit word) and the strong flag of the component
  unsigned long long lo = 0, hi = 0;
  {
    int j = 0;
    for (unsigned rem = emask; rem; j++) {
      const unsigned low = rem & (0u - rem), x = rem + low, rm = rem & ~x;
      rem &= x;
      const unsigned c = num[uf_find_ro(lab, s0 + j)];      // (after the flattening: one or two hops)
      if (j < 8) lo |= (unsigned long long)c << (8 * j); else hi |= (unsigned long long)c << (8 * (j - 8));
      if (smask & rm) cst[c] = 1;
    }
  }
  unsigned char *dst = runc + ((size_t)tile * HT + lane) * HYST_MAX_RUNS;   // only the words that hold runs
  if (nr > 8) *reinterpret_cast<uint4 *>(dst) = make_uint4((unsigned)lo, (unsigned)(lo >> 32), (unsigned)hi, (unsigned)(hi >> 32));
  else if (nr > 4) *reinterpret_cast<uint2 *>(dst) = make_uint2((unsigned)lo, (unsigned)(lo >> 32));
  else if (nr > 0) *reinterpret_cast<unsigned *>(dst) = (unsigned)lo;
  __syncwarp();
  const int id0 = HYST_MAX_ROOTS * tile;
  for (int c = lane; c < total; c += 32) { parent[id0 + c] = id0 + c; strong[id0 + c] = cst[c]; }
  if (lane == 0) ncomp[tile] = total;
}

// The component number of the j-th run of row r of tile t, as hyst_local_kernel stored it (j < runs of the row).
__device__ __forceinline__ unsigned run_comp(const unsigned char *__restrict__ runc, int t, int r, int j) {
  return runc[((size_t)t * HT + r) * HYST_MAX_RUNS + j];
}
// Component id of the edge pixel (x, r) of tile t.
__device__ __forceinline__ int pixel_comp(const unsigned *__restrict__ E, const unsigned char *__restrict__ runc, int t, int r, int x) {
  return HYST_MAX_ROOTS * t + (int)run_comp(runc, t, r, run_ordinal(__ldg(E + (size_t)HT * t + r), x));
}
// Unions across one seam.  a, b: the pixels on either side of it as bit masks along the seam (bit i of a touches
// bits i-1 .. i+1 of b).  Consecutive set bits of one side are 8-connected, hence one component of their tile:
// the lane that holds the first bit of a run of `a` links that run to every run of `b` it touches.
template <class IdA, class IdB>
__device__ __forceinline__ void seam_union(int *parent, unsigned a, unsigned b, int lane, IdA ida, IdB idb) {
  if (!((a >> lane) & 1u) || (lane > 0 && ((a >> (lane - 1)) & 1u))) return;
  const unsigned rm = run_mask_from(a, lane);
  unsigned touch = b & (rm | (rm << 1) | (rm >> 1));
  if (!touch) return;
  const int me = ida(lane);
  do {
    const int us = run_start(b, __ffs(touch) - 1);
    const unsigned uhi = b >> us << us;
    touch &= ~(uhi & ~(uhi + (1u << us)));
    uf_union(parent, me, idb(us));
  } while (touch);
}
// Seams.  ONE WARP per tile (8 tiles per CTA): its right seam (column 31 against column 0 of the right tile), its
// bottom seam (row 31 against row 0 of the tile below) and its two lower diagonal corners; every pair of
// neighbouring tiles is thus visited once.
__global__ void __launch_bounds__(256)
hyst_seam_kernel(const unsigned *__restrict__ E, const unsigned char *__restrict__ runc, int *__restrict__ parent,
                 int TX, int TY, int n_tiles) {
  const int lane = threadIdx.x & 31;
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (t >= n_tiles) return;
  const unsigned row = E[(size_t)HT * t + lane];
  if (!__any_sync(0xffffffffu, row != 0)) return;
  const int tx = t % TX, ty = (t / TX) % TY;
  const unsigned last = __shfl_sync(0xffffffffu, row, HT - 1);
  if (tx + 1 < TX) {
    const int tr = t + 1;
    const unsigned col_a = __ballot_sync(0xffffffffu, row >> (HT - 1));
    const unsigned col_b = __ballot_sync(0xffffffffu, E[(size_t)HT * tr + lane] & 1u);
    seam_union(parent, col_a, col_b, lane, [&](int r) { return pixel_comp(E, runc, t, r, HT - 1); },
               [&](int r) { return HYST_MAX_ROOTS * tr + (int)run_comp(runc, tr, r, 0); });
  }
  if (ty + 1 < TY) {
    const int tb = t + TX;
    const unsigned first = __ldg(E + (size_t)HT * tb);
    seam_union(parent, last, first, lane, [&](int x) { return pixel_comp(E, runc, t, HT - 1, x); },
               [&](int x) { return pixel_comp(E, runc, tb, 0, x); });
    if (lane == 0) {
      if (tx + 1 < TX && (last >> (HT - 1)) && (__ldg(E + (size_t)HT * (tb + 1)) & 1u))
        uf_union(parent, pixel_comp(E, runc, t, HT - 1, HT - 1), HYST_MAX_ROOTS * (tb + 1) + (int)run_comp(runc, tb + 1, 0, 0));
      if (tx > 0 && (last & 1u) && (__ldg(E + (size_t)HT * (tb - 1)) >> (HT - 1)))
        uf_union(parent, HYST_MAX_ROOTS * t + (int)run_comp(runc, t, HT - 1, 0), pixel_comp(E, runc, tb - 1, 0, HT - 1));
    }
  }
}
// A component that holds a class-2 pixel marks its global root.  One warp per tile walks the tile's components.
__global__ void __launch_bounds__(256)
hyst_mark_kernel(const int *__restrict__ ncomp, int *__restrict__ parent, unsigned char *strong, int n_tiles) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const int n = ncomp[t];
  for (int c = lane; c < n; c += 32) {
    const int id = HYST_MAX_ROOTS * t + c;
    if (strong[id]) strong[uf_find(parent, id)] = 1;
  }
}
// Every component learns whether its global component holds a class-2 pixel.
__global__ void __launch_bounds__(256)
hyst_resolve_kernel(const int *__restrict__ ncomp, int *__restrict__ parent, const unsigned char *__restrict__ strong,
                    unsigned char *__restrict__ keep, int n_tiles) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= n_tiles) return;
  const int n = ncomp[t];
  for (int c = lane; c < n; c += 32) {
    const int id = HYST_MAX_ROOTS * t + c;
    keep[id] = strong[uf_find(parent, id)];
  }
}
// Edge map.  ONE WARP per tile (8 tiles per CTA), lane r on row r: the runs of the row whose component is kept
// form the output word.  The CTA then writes its 8 tiles row by row, 32 bytes 0 / 255 per tile row and thread, so
// that a warp stores 4 rows of 8 neighbouring tiles (every pixel of the image, empty tiles included).  One
// atomicAdd per frame and CTA into the edge-pixel count.
__global__ void __launch_bounds__(256)
hyst_emit_kernel(const unsigned *__restrict__ E, const unsigned char *__restrict__ runc, const unsigned char *__restrict__ keep,
                 unsigned char *__restrict__ edges, int *__restrict__ nonzero, int nx, int ny, int TX, int TY, int n_tiles, int vec) {
  __shared__ int s_cnt[8], s_f[8];
  __shared__ unsigned s_out[8][HT];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int t = blockIdx.x * 8 + warp;
  int cnt = 0, f = -1;
  if (t < n_tiles) {
    f = t / (TX * TY);
    const unsigned bits = E[(size_t)HT * t + lane];
    unsigned out = 0;
    if (bits) {
      const int nr = __popc(bits & ~(bits << 1));
      const unsigned char *src = runc + ((size_t)t * HT + lane) * HYST_MAX_RUNS;   // the words hyst_local_kernel wrote
      uint4 w = make_uint4(0, 0, 0, 0);
      if (nr > 8) w = *reinterpret_cast<const uint4 *>(src);
      else if (nr > 4) { const uint2 h = *reinterpret_cast<const uint2 *>(src); w.x = h.x; w.y = h.y; }
      else w.x = *reinterpret_cast<const unsigned *>(src);
      const unsigned char *kp = keep + HYST_MAX_ROOTS * t;
      int j = 0;
      for (unsigned rem = bits; rem; j++) {
        const unsigned low = rem & (0u - rem), x = rem + low, rm = rem & ~x;
        rem &= x;
        const unsigned word = j < 4 ? w.x : j < 8 ? w.y : j < 12 ? w.z : w.w;
        if (kp[(word >> (8 * (j & 3))) & 0xffu]) out |= rm;
      }
    }
    cnt = __popc(out);
    s_out[warp][lane] = out;
  }
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) { s_cnt[warp] = cnt; s_f[warp] = f; }
  __syncthreads();
  {
    const int w = threadIdx.x & 7, r = threadIdx.x >> 3, tw = blockIdx.x * 8 + w;
    const int tx = tw % TX, ty = (tw / TX) % TY, gy = ty * HT + r, gx = tx * HT;
    if (tw < n_tiles && gy < ny) {
      const unsigned out = s_out[w][r];
      unsigned char *dst = edges + ((size_t)s_f[w] * ny + gy) * nx + gx;
      if (vec && gx + HT <= nx) {
        unsigned o[8];
#pragma unroll
        for (int q = 0; q < 8; q++) o[q] = (((out >> (4 * q)) & 0xfu) * 0x00204081u & 0x01010101u) * 0xffu;   // 4 bits -> 4 bytes
        reinterpret_cast<uint4 *>(dst)[0] = make_uint4(o[0], o[1], o[2], o[3]);
        reinterpret_cast<uint4 *>(dst)[1] = make_uint4(o[4], o[5], o[6], o[7]);
      } else {
        for (int x = 0; x < HT && gx + x < nx; x++) dst[x] = ((out >> x) & 1u) ? 255 : 0;
      }
    }
  }
  if (threadIdx.x == 0) {                    // the 8 tiles may span two (or, for tiny frames, more) frames
    int acc = 0, cf = s_f[0];
    for (int w = 0; w < 8; w++) {
      if (s_f[w] != cf) { if (cf >= 0 && acc) atomicAdd(&nonzero[cf], acc); acc = 0; cf = s_f[w]; }
      acc += s_cnt[w];
    }
    if (cf >= 0 && acc) atomicAdd(&nonzero[cf], acc);
  }
}

// Class bytes -> the tile-major masks E, S that canny_grad_nms_spec2_kernel writes (b2f_canny_hysteresis_dev only).
// Same grid as the NMS kernel, one ballot pair per tile row; pixels outside the image give 0 bits.
__global__ void __launch_bounds__(256)
hyst_pack_kernel(const unsigned char *__restrict__ cls, unsigned *__restrict__ emask, unsigned *__restrict__ smask, int nx, int ny) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int gx = blockIdx.x * HT + lane;
  const unsigned char *src = cls + (size_t)blockIdx.z * nx * ny;
  const size_t t = ((size_t)blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
#pragma unroll
  for (int k = 0; k < HT / 8; k++) {
    const int ly = warp + 8 * k, gy = blockIdx.y * HT + ly;
    const unsigned char c = (gx < nx && gy < ny) ? __ldg(src + (size_t)gy * nx + gx) : (unsigned char)0;
    const unsigned e = __ballot_sync(0xffffffffu, c != 0), s = __ballot_sync(0xffffffffu, c == 2);
    if (lane == 0) { emask[HT * t + ly] = e; smask[HT * t + ly] = s; }
  }
}

// ------------------------------------------------------------------------------------------ host
// tap list of one axis: orc_canny_taps restated (tools.c:146-163): wrap coordinates, exp(-c^2/s^2),
// unit sum over the full period, taps below 2^-64 dropped.
static void make_taps(int w, double s, std::vector<int> &coord, std::vector<double> &weight) {
  double inv_s = 1 / s, total = 0;
  for (int i = 0; i < w; i++) { double c = i < w / 2 ? i : i - w; total += exp(-c * c * inv_s * inv_s); }
  int lo = -(w - w / 2), hi = w / 2 - 1;
  coord.clear(); weight.clear();
  for (int c = lo; c <= hi; c++) {
    double g = exp(-(double)c * c * inv_s * inv_s);
    if (g < 0x1p-64) continue;
    coord.push_back(c); weight.push_back(g / total);
  }
}
static bool symmetric_taps(const std::vector<int> &c, const std::vector<double> &w, CannyTaps &out) {
  int n = (int)c.size();
  if (n % 2 == 0) return false;
  int R = n / 2;
  if (R > CANNY_MAXR) return false;
  for (int k = 0; k <= R; k++) {
    if (c[R - k] != -k || c[R + k] != k || w[R - k] != w[R + k]) return false;
    out.w[k] = w[R + k];
  }
  out.R = R;
  return true;
}

// Scratch of the hysteresis stage for `tiles` 32x32 tiles, the edge and strong masks included.
static size_t hyst_scratch_bytes(size_t tiles) {
  return 2 * align256(tiles * HT * 4) /*edge, strong masks*/ + align256(tiles * HT * HYST_MAX_RUNS) /*runc*/ +
         align256(tiles * 4) /*ncomp*/ + align256(tiles * HYST_MAX_ROOTS * 4) /*parent*/ + 2 * align256(tiles * HYST_MAX_ROOTS) /*strong, keep*/;
}
static size_t hyst_tile_count(int n_frames, int nx, int ny) { return (size_t)ceil_div(nx, HT) * ceil_div(ny, HT) * n_frames; }

size_t canny_scratch_bytes(int n_frames, int nx, int ny) {
  const size_t n = (size_t)n_frames * nx * ny;
  return align256(n * 4) /*blur*/ + hyst_scratch_bytes(hyst_tile_count(n_frames, nx, ny)) +
         align256(n * 8) /*blur row sums (generic path rows)*/ + (1 << 16) /*generic path tap lists*/;
}

// The batch limits of the Canny path: pixel offsets and the component ids 256*tile + c of the hysteresis are int.
static int canny_batch_geometry(const char *who, int n_frames, int nx, int ny, int *TX, int *TY, int *n_tiles) {
  if ((size_t)nx * ny * n_frames >= (size_t)1 << 31) {
    set_error("%s: batch of %d frames %dx%d exceeds 2^31 pixels; split the batch", who, n_frames, nx, ny);
    return B2F_EUNSUP;
  }
  const size_t tiles = hyst_tile_count(n_frames, nx, ny);
  if (tiles * HYST_MAX_ROOTS >= (size_t)1 << 31) {   // (only very thin frames get here)
    set_error("%s: batch of %d frames %dx%d has too many 32x32 tiles; split the batch", who, n_frames, nx, ny);
    return B2F_EUNSUP;
  }
  *TX = ceil_div(nx, HT); *TY = ceil_div(ny, HT); *n_tiles = (int)tiles;
  return B2F_OK;
}

// Hysteresis on the tile-major masks emask / smask of n_frames frames (TX x TY tiles each): the edge map (0 / 255) to
// d_edges and the number of edge pixels per frame to d_nonzero.  Carves its scratch (hyst_scratch_bytes less the masks)
// from the arena.  Per-component arrays are written by hyst_local for the ids that exist: no memsets.
static int canny_hysteresis(b2f_ctx *ctx, const unsigned *emask, const unsigned *smask, int n_frames, int nx, int ny, int TX,
                            int TY, int n_tiles, unsigned char *d_edges, int *d_nonzero, cudaStream_t st) {
  const size_t tiles = (size_t)n_tiles;
  unsigned char *runc = ctx->arena.get<unsigned char>(tiles * HT * HYST_MAX_RUNS);
  int *ncomp = ctx->arena.get<int>(tiles);
  int *parent = ctx->arena.get<int>(tiles * HYST_MAX_ROOTS);
  unsigned char *strong = ctx->arena.get<unsigned char>(tiles * HYST_MAX_ROOTS), *keep = ctx->arena.get<unsigned char>(tiles * HYST_MAX_ROOTS);
  B2F_ARENA_CHECK(ctx);
  B2F_CUDA(cudaMemsetAsync(d_nonzero, 0, sizeof(int) * n_frames, st));
  const unsigned hb = (unsigned)ceil_div(n_tiles, 8);
  hyst_local_kernel<<<hb, 256, 0, st>>>(emask, smask, runc, ncomp, parent, strong, n_tiles);
  B2F_LAUNCH_CHECK(ctx);
  hyst_seam_kernel<<<hb, 256, 0, st>>>(emask, runc, parent, TX, TY, n_tiles);
  B2F_LAUNCH_CHECK(ctx);
  hyst_mark_kernel<<<hb, 256, 0, st>>>(ncomp, parent, strong, n_tiles);
  B2F_LAUNCH_CHECK(ctx);
  hyst_resolve_kernel<<<hb, 256, 0, st>>>(ncomp, parent, strong, keep, n_tiles);
  B2F_LAUNCH_CHECK(ctx);
  const int vec = (nx % 16 == 0) && ((reinterpret_cast<uintptr_t>(d_edges) & 15) == 0);
  hyst_emit_kernel<<<hb, 256, 0, st>>>(emask, runc, keep, d_edges, d_nonzero, nx, ny, TX, TY, n_tiles, vec);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

int canny_device(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, int nx, int ny, double s, double low_thr,
                 double high_thr, int acc_grad, unsigned char *d_edges, int *d_nonzero, cudaStream_t st) {
  const size_t n = (size_t)nx * ny * n_frames;
  int TX, TY, n_tiles;
  int rc = canny_batch_geometry("canny", n_frames, nx, ny, &TX, &TY, &n_tiles);
  if (rc != B2F_OK) return rc;
  if (!(s > 0)) { set_error("canny: s must be > 0"); return B2F_EINVAL; }
  const size_t tiles = (size_t)n_tiles;
  float *blur = ctx->arena.get<float>(n);
  unsigned *emask = ctx->arena.get<unsigned>(tiles * HT), *smask = ctx->arena.get<unsigned>(tiles * HT);
  std::vector<int> cx, cy; std::vector<double> wx, wy;
  make_taps(nx, s, cx, wx); make_taps(ny, s, cy, wy);
  CannyTaps tx, ty;
  const bool sym = symmetric_taps(cx, wx, tx) && symmetric_taps(cy, wy, ty);   // same rule as the oracle (R <= 64)
  size_t smem = 0;
  if (sym) smem = sizeof(double) * ((size_t)(CB_TH + 2 * ty.R) * CB_TW + (size_t)(CB_TH + 2 * ty.R) * ((CB_TW + 2 * tx.R + 1) & ~1));
  if (sym && smem <= 200 * 1024) {
    B2F_ARENA_CHECK(ctx);
    dim3 grid(ceil_div(nx, CB_TW), ceil_div(ny, CB_TH), n_frames);
    static const bool tiled13 = getenv("B2F_CANNY_TILED_BLUR") != nullptr;
    if (tx.R == 13 && ty.R == 13 && !tiled13 && nx >= 64 && ny >= 64) {
      // two-kernel variant: row sums (doubles) go through HBM/L2 once, no halo recomputation
      double *rowsum = ctx->arena.get<double>(n);
      B2F_ARENA_CHECK(ctx);
      canny_blur_rows_kernel<13><<<dim3(ceil_div(ceil_div(nx, 4), 256), ny, n_frames), 256, 0, st>>>(d_frames, rowsum, nx, ny, tx);
      B2F_LAUNCH_CHECK(ctx);
      const size_t csm = sizeof(double) * (size_t)(CC_TH + 26) * CC_TW;
      // function attributes are per device: set on every launch, never cached per process
      B2F_CUDA(cudaFuncSetAttribute(canny_blur_cols_kernel<13>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)csm));
      canny_blur_cols_kernel<13><<<dim3(ceil_div(nx, CC_TW), ceil_div(ny, CC_TH), n_frames), 256, csm, st>>>(rowsum, blur, nx, ny, ty);
    } else if (tx.R == 13 && ty.R == 13) {
      B2F_CUDA(cudaFuncSetAttribute(canny_blur_kernel<13>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      canny_blur_kernel<13><<<grid, CB_NT, smem, st>>>(d_frames, blur, nx, ny, tx, ty);
    } else {
      B2F_CUDA(cudaFuncSetAttribute(canny_blur_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      canny_blur_kernel<0><<<grid, CB_NT, smem, st>>>(d_frames, blur, nx, ny, tx, ty);
    }
    B2F_LAUNCH_CHECK(ctx);
  } else {
    double *tmp = ctx->arena.get<double>(n);
    int *dcx = ctx->arena.get<int>(cx.size() + cy.size());
    double *dwx = ctx->arena.get<double>(wx.size() + wy.size());
    B2F_ARENA_CHECK(ctx);
    B2F_CUDA(cudaMemcpyAsync(dcx, cx.data(), cx.size() * 4, cudaMemcpyHostToDevice, st));
    B2F_CUDA(cudaMemcpyAsync(dcx + cx.size(), cy.data(), cy.size() * 4, cudaMemcpyHostToDevice, st));
    B2F_CUDA(cudaMemcpyAsync(dwx, wx.data(), wx.size() * 8, cudaMemcpyHostToDevice, st));
    B2F_CUDA(cudaMemcpyAsync(dwx + wx.size(), wy.data(), wy.size() * 8, cudaMemcpyHostToDevice, st));
    B2F_CUDA(cudaStreamSynchronize(st));   // host vectors go out of scope below
    dim3 grid(ceil_div(nx, 128), ny, n_frames);
    canny_blur_generic_rows<<<grid, 128, 0, st>>>(d_frames, tmp, nx, ny, TapList{dcx, dwx, (int)cx.size(), sym ? 1 : 0});
    B2F_LAUNCH_CHECK(ctx);
    canny_blur_generic_cols<<<grid, 128, 0, st>>>(tmp, blur, nx, ny, TapList{dcx + cx.size(), dwx + wx.size(), (int)cy.size(), sym ? 1 : 0});
    B2F_LAUNCH_CHECK(ctx);
  }
  // pixels sent to the exact tier since the context was created (one atomicAdd per tile that has any): b2f_canny_stats
  if (!ctx->canny_stats) {
    B2F_CUDA(cudaMalloc(&ctx->canny_stats, 8));
    B2F_CUDA(cudaMemsetAsync(ctx->canny_stats, 0, 8, st));
  }
  unsigned long long *fc = static_cast<unsigned long long *>(ctx->canny_stats);
  // thresholds truncate like rcpp_canny.cpp:180
  if (acc_grad)
    canny_grad_nms_spec2_kernel<true><<<dim3(TX, TY, n_frames), CG_NT, 0, st>>>(blur, emask, smask, nx, ny, (int)low_thr, (int)high_thr, fc);
  else
    canny_grad_nms_spec2_kernel<false><<<dim3(TX, TY, n_frames), CG_NT, 0, st>>>(blur, emask, smask, nx, ny, (int)low_thr, (int)high_thr, fc);
  B2F_LAUNCH_CHECK(ctx);
  return canny_hysteresis(ctx, emask, smask, n_frames, nx, ny, TX, TY, n_tiles, d_edges, d_nonzero, st);
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_canny_stats(b2f_ctx *ctx, unsigned long long *tier2_pixels) {
  if (!ctx || !tier2_pixels) { set_error("b2f_canny_stats: NULL argument"); return B2F_EINVAL; }
  *tier2_pixels = 0;
  if (!ctx->canny_stats) return B2F_OK;
  B2F_CUDA(cudaSetDevice(ctx->device));
  B2F_CUDA(cudaMemcpyAsync(tier2_pixels, ctx->canny_stats, 8, cudaMemcpyDeviceToHost, ctx->stream));
  B2F_CUDA(cudaStreamSynchronize(ctx->stream));
  return B2F_OK;
}

int b2f_canny_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int nx, int ny, double s, double low_thr,
                  double high_thr, int acc_grad, uint8_t *d_edges, int *d_nonzero, void *stream) {
  if (!ctx || !d_frames || !d_edges || !d_nonzero || n_frames <= 0 || nx <= 0 || ny <= 0) { set_error("b2f_canny_dev: bad argument"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  int rc = stream_handoff(ctx, stream, &st);
  if (rc != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, canny_scratch_bytes(n_frames, nx, ny))) != B2F_OK) return rc;
  return canny_device(ctx, d_frames, n_frames, nx, ny, s, low_thr, high_thr, acc_grad, d_edges, d_nonzero, st);
}

int b2f_canny_hysteresis_dev(b2f_ctx *ctx, const uint8_t *d_cls, int n_frames, int nx, int ny, uint8_t *d_edges,
                             int *d_nonzero, void *stream) {
  if (!ctx || !d_cls || !d_edges || !d_nonzero || n_frames <= 0 || nx <= 0 || ny <= 0) { set_error("b2f_canny_hysteresis_dev: bad argument"); return B2F_EINVAL; }
  int TX, TY, n_tiles;
  int rc = canny_batch_geometry("b2f_canny_hysteresis_dev", n_frames, nx, ny, &TX, &TY, &n_tiles);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, hyst_scratch_bytes((size_t)n_tiles))) != B2F_OK) return rc;
  unsigned *emask = ctx->arena.get<unsigned>((size_t)n_tiles * HT), *smask = ctx->arena.get<unsigned>((size_t)n_tiles * HT);
  B2F_ARENA_CHECK(ctx);
  hyst_pack_kernel<<<dim3(TX, TY, n_frames), 256, 0, st>>>(d_cls, emask, smask, nx, ny);
  B2F_LAUNCH_CHECK(ctx);
  return canny_hysteresis(ctx, emask, smask, n_frames, nx, ny, TX, TY, n_tiles, d_edges, d_nonzero, st);
}

int b2f_canny_batch(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int nx, int ny, double s, double low_thr,
                    double high_thr, int acc_grad, uint8_t *edges, int *nonzero) {
  if (!ctx || !frames || !edges || !nonzero || n_frames <= 0 || nx <= 0 || ny <= 0) { set_error("b2f_canny_batch: bad argument"); return B2F_EINVAL; }
  const b2f_canny_params cp = {s, low_thr, high_thr, acc_grad};
  return features_batch("b2f_canny_batch", ctx, frames, 1, n_frames, ny, nx, nullptr, 0, nullptr, nullptr, nullptr, nullptr,
                        &cp, edges, nonzero, 0, 0, 0, nullptr);
}

int b2f_canny_host(b2f_ctx *ctx, const uint8_t *img, int nx, int ny, double s, double low_thr, double high_thr,
                   int acc_grad, uint8_t *edges, int *nonzero) {
  return b2f_canny_batch(ctx, img, 1, nx, ny, s, low_thr, high_thr, acc_grad, edges, nonzero);
}

}  // extern "C"
