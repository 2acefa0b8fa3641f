// harris.cu — host orchestration + remaining kernels of the Harris corner path
// (image.CornerDetectionHarris; SURVEY.md §8a rows H1-H7).
//
//   response map    harris_fused3_kernel (harris_kernels3.cuh) or the bit-exact staged kernels here
//   NMS             nms_bitmask_kernel: window predicate of harris.cpp:141-255 -> 1 bit / pixel
//   compaction      row_count / row_scan / emit kernels -> corners in raster order (harris.cpp:250-252)
//   certification   nms_tolerant_kernel (candidates of the fp32 map with its error bound) ->
//                   harris_exact_patch_kernel (reference arithmetic on a patch) -> compact_kept_kernel:
//                   the fast path's key-point lists and strengths are the reference's, bit for bit
//   selection, sub-pixel, scale check (H7, <1 % of the time): harris_api.cu
#include "harris_kernels3.cuh"
#include "harris_host.h"
#include <cmath>
#include <algorithm>

namespace b2f {

// ------------------------------------------------------------------------------------------
// bit-exact staged kernels (reference operation order, no FMA contraction)
// ------------------------------------------------------------------------------------------
struct ExactTaps { double B[HARRIS_MAX_TAPS]; int size; };

__device__ __forceinline__ int pad_index(int p, int n) {   // gaussian.cpp:345-349
  if (p < 0) return -p;
  if (p >= n) return 2 * n - 1 - p;
  return p;
}

// one pass of discrete_gaussian (gaussian.cpp:332-361 rows / :363-392 columns)
template <bool COLS>
__global__ void exact_gauss_pass(const float *__restrict__ src, float *__restrict__ dst, int nx, int ny,
                                 const __grid_constant__ ExactTaps tp) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= nx) return;
  size_t plane = (size_t)nx * ny * blockIdx.z;
  const float *s = src + plane;
  const int n = COLS ? ny : nx, i = COLS ? y : x;
  auto at = [&](int q) -> double {
    int p = pad_index(q, n);
    return (double)(COLS ? s[(size_t)p * nx + x] : s[(size_t)y * nx + p]);
  };
  double sum = __dmul_rn(tp.B[0], at(i));
  for (int j = 1; j < tp.size; j++) sum = __dadd_rn(sum, __dmul_rn(tp.B[j], __dadd_rn(at(i - j), at(i + j))));
  dst[plane + (size_t)y * nx + x] = __double2float_rn(sum);
}

// SII 1-D pass, one thread per line, sequential float running sum (gaussian.cpp:179-215)
struct SiiCoef { float w[3]; int r[3]; };
__global__ void exact_sii_pass(const float *__restrict__ src, float *__restrict__ dst, float *__restrict__ scratch,
                               int nx, int ny, int cols, SiiCoef c) {
  int line = blockIdx.x * blockDim.x + threadIdx.x;
  int nlines = cols ? nx : ny;
  if (line >= nlines) return;
  size_t plane = (size_t)nx * ny * blockIdx.y;
  const int n = cols ? ny : nx;
  const size_t stride = cols ? nx : 1;
  const float *s = src + plane + (cols ? (size_t)line : (size_t)line * nx);
  float *d = dst + plane + (cols ? (size_t)line : (size_t)line * nx);
  const int pad = c.r[0] + 1;
  const int nmax = nx > ny ? nx : ny;
  float *b = scratch + ((size_t)blockIdx.y * nmax + line) * (size_t)(nmax + 2 * pad) + pad;
  float acc = 0.f;
  for (int i = -pad; i < n + pad; i++) {
    int q = i < 0 ? 0 : (i >= n ? n - 1 : i);
    acc = __fadd_rn(acc, s[stride * q]);
    b[i] = acc;
  }
  for (int i = 0; i < n; i++) {
    float a = __fmul_rn(c.w[0], __fsub_rn(b[i + c.r[0]], b[i - c.r[0] - 1]));
    a = __fadd_rn(a, __fmul_rn(c.w[1], __fsub_rn(b[i + c.r[1]], b[i - c.r[1] - 1])));
    a = __fadd_rn(a, __fmul_rn(c.w[2], __fsub_rn(b[i + c.r[2]], b[i - c.r[2] - 1])));
    d[stride * i] = a;
  }
}

// gradient (gradient.cpp:17-128) + products (harris.cpp:57-62), exact float roundings
__global__ void exact_grad_products(const float *__restrict__ Is, float *__restrict__ A, float *__restrict__ B,
                                    float *__restrict__ C, int nx, int ny, int grad) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= nx) return;
  size_t plane = (size_t)nx * ny * blockIdx.z;
  const float *I = Is + plane;
  int cx = min(max(x, 1), nx - 2), cy = min(max(y, 1), ny - 2);   // replicate rule, gradient.cpp:40-55
  size_t p = (size_t)cy * nx + cx;
  float ix, iy;
  if (grad == 1) {
    float hx = __fsub_rn(I[p + 1], I[p - 1]);
    float dx = __fsub_rn(__fsub_rn(__fadd_rn(I[p - nx + 1], I[p + nx + 1]), I[p - nx - 1]), I[p + nx - 1]);
    ix = __double2float_rn(__dadd_rn(__dmul_rn(0.25, (double)hx), __dmul_rn(0.125, (double)dx)));
    float hy = __fsub_rn(I[p + nx], I[p - nx]);
    float dy = __fsub_rn(__fsub_rn(__fadd_rn(I[p + nx + 1], I[p + nx - 1]), I[p - nx + 1]), I[p - nx - 1]);
    iy = __double2float_rn(__dadd_rn(__dmul_rn(0.25, (double)hy), __dmul_rn(0.125, (double)dy)));
  } else {
    ix = __fmul_rn(0.5f, __fsub_rn(I[p + 1], I[p - 1]));
    iy = __fmul_rn(0.5f, __fsub_rn(I[p + nx], I[p - nx]));
  }
  size_t o = plane + (size_t)y * nx + x;
  A[o] = __fmul_rn(ix, ix); B[o] = __fmul_rn(ix, iy); C[o] = __fmul_rn(iy, iy);
}

__global__ void exact_response(const float *__restrict__ A, const float *__restrict__ B, const float *__restrict__ C,
                               float *__restrict__ R, size_t n, float k, int measure) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) R[i] = corner_measure(A[i], B[i], C[i], k, measure);
}

__global__ void u8_to_float(const unsigned char *__restrict__ s, float *__restrict__ d, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = (float)s[i];
}

// zoom_out (zoom.cpp:121-139): bicubic sampled at even integer positions == decimation
__global__ void decimate2(const float *__restrict__ s, float *__restrict__ d, int nx, int ny) {
  int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  int nxx = nx / 2, nyy = ny / 2;
  if (x < nxx && y < nyy) d[(size_t)y * nxx + x] = s[(size_t)(2 * y) * nx + 2 * x];
}

// ------------------------------------------------------------------------------------------
// NMS: window predicate -> bitmask
//   (x,y) in [r,n-r), R>=Th, strictly greater than every window value in rows above and
//   same-row values to the right, >= same-row values to the left and rows below
//   (harris.cpp:170-243 restated order-free; SURVEY.md §8a-H6).
// ------------------------------------------------------------------------------------------
constexpr int NMS_TW = 128, NMS_TH = 16, NMS_NT = 256;

__global__ void __launch_bounds__(NMS_NT)
nms_bitmask_kernel(const float *__restrict__ R, unsigned *__restrict__ mask, int nx, int ny, int words_per_row,
                   float Th, int radius) {
  extern __shared__ float tile[];
  const int P = NMS_TW + 2 * radius;           // tile pitch
  const int TH2 = NMS_TH + 2 * radius;
  const int x0 = blockIdx.x * NMS_TW, y0 = blockIdx.y * NMS_TH;
  const float *Rf = R + (size_t)nx * ny * blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;    // 8 warps
  for (int r = warp; r < TH2; r += NMS_NT / 32) {                // a warp streams whole tile rows
    const int gy = y0 - radius + r;
    const bool rowok = gy >= 0 && gy < ny;
    const float *src = Rf + (size_t)(rowok ? gy : 0) * nx;
    for (int c = lane; c < P; c += 32) {
      const int gx = x0 - radius + c;
      tile[r * P + c] = (rowok && gx >= 0 && gx < nx) ? __ldg(src + gx) : -INFINITY;
    }
  }
  __syncthreads();
#pragma unroll 1
  for (int s = warp; s < NMS_TH * (NMS_TW / 32); s += NMS_NT / 32) {
    int row = s / (NMS_TW / 32), seg = s - row * (NMS_TW / 32);
    int lx = seg * 32 + lane, gx = x0 + lx, gy = y0 + row;
    const float *c = tile + (row + radius) * P + lx + radius;
    float v = *c;
    bool ok = gx >= radius && gx < nx - radius && gy >= radius && gy < ny - radius && !(v < Th);
    if (ok) {   // cheap 3x3 pre-test, then the full window
      ok = v > c[-P - 1] && v > c[-P] && v > c[-P + 1] && v > c[1] && v >= c[-1] && v >= c[P - 1] && v >= c[P] && v >= c[P + 1];
      if (gx == radius && c[-1] >= v) ok = false;   // the row scan starts by walking off the downhill (harris.cpp:173)
    }
    if (ok) {
      for (int dy = -radius; dy <= radius && ok; dy++) {
        const float *q = c + dy * P;
        if (dy < 0) { for (int dx = -radius; dx <= radius; dx++) ok = ok && (v > q[dx]); }
        else if (dy > 0) { for (int dx = -radius; dx <= radius; dx++) ok = ok && (v >= q[dx]); }
        else {
          for (int dx = -radius; dx < 0; dx++) ok = ok && (v >= q[dx]);
          for (int dx = 1; dx <= radius; dx++) ok = ok && (v > q[dx]);
        }
      }
    }
    unsigned bits = __ballot_sync(0xffffffffu, ok);
    int word = (x0 >> 5) + seg;
    if (lane == 0 && gy < ny && word < words_per_row)
      mask[((size_t)blockIdx.z * ny + gy) * words_per_row + word] = bits;
  }
}

// The row scan of harris.cpp:170-243 begins by walking down the leading run of the row (:175-176): it passes over every
// pixel that is below the threshold, marked by the rows above, or not above its left neighbour.  A window maximum is passed
// over only if its left neighbour ties it exactly, and then whether the walk gets there depends on the whole row prefix
// and on the marks of the rows above.  The window predicate settles x == radius only.  One block per frame looks for any
// other kept pixel tied with its left neighbour — exact ties at a maximum are rare: plateaus, or ridges of equal values
// along straight edges when k < 0 — and, if there is one, one thread scans the frame again in the reference's order with
// its skip mask and rewrites the frame's list and count.
__global__ void __launch_bounds__(256)
nms_tie_rescan_kernel(const float *__restrict__ R, const unsigned *__restrict__ mask, unsigned char *__restrict__ skip_all,
                      int nx, int ny, int words_per_row, float Th, int radius, int cap, int *__restrict__ xy,
                      float *__restrict__ strength, int *__restrict__ counts) {
  __shared__ int tie;
  const int f = blockIdx.x;
  const size_t plane = (size_t)nx * ny;
  const float *Rf = R + (size_t)f * plane;
  const unsigned *mf = mask + (size_t)f * ny * words_per_row;
  if (threadIdx.x == 0) tie = 0;
  __syncthreads();
  for (size_t w = threadIdx.x; w < (size_t)ny * words_per_row; w += blockDim.x) {
    unsigned bits = mf[w];
    const int y = (int)(w / words_per_row), x0 = (int)(w % words_per_row) * 32;
    while (bits) {
      const int x = x0 + __ffs(bits) - 1;
      bits &= bits - 1;
      if (x > radius && Rf[(size_t)y * nx + x - 1] == Rf[(size_t)y * nx + x]) tie = 1;
    }
  }
  __syncthreads();
  if (!tie) return;
  unsigned char *skip = skip_all + (size_t)f * plane;
  for (size_t i = threadIdx.x; i < plane; i += blockDim.x) skip[i] = Rf[i] < Th;
  __syncthreads();
  if (threadIdx.x != 0) return;
  int count = 0;
  for (int i = radius; i < ny - radius; i++) {
    const float *row = Rf + (size_t)i * nx;
    unsigned char *srow = skip + (size_t)i * nx;
    int j = radius;
    while (j < nx - radius && (srow[j] || row[j - 1] >= row[j])) j++;
    while (j < nx - radius) {
      while (j < nx - radius && (srow[j] || row[j + 1] >= row[j])) j++;
      if (j >= nx - radius) break;
      int p1 = j + 2;                                          // right of the peak: smaller values are marked
      while (p1 <= j + radius && row[p1] < row[j]) { srow[p1] = 1; p1++; }
      if (p1 > j + radius) {
        int p2 = j - 1;                                        // left: ties allowed
        while (p2 >= j - radius && row[p2] <= row[j]) p2--;
        if (p2 < j - radius) {
          bool found = false;
          for (int k = i + radius; !found && k > i; k--)        // rows below, backwards: values not above are marked
            for (int l = j + radius; !found && l >= j - radius; l--) {
              if (Rf[(size_t)k * nx + l] > row[j]) found = true;
              else skip[(size_t)k * nx + l] = 1;
            }
          for (int k = i - radius; !found && k < i; k++)        // rows above: ties end it
            for (int l = j - radius; !found && l <= j + radius; l++)
              if (Rf[(size_t)k * nx + l] >= row[j]) found = true;
          if (!found) {
            if (count < cap) { xy[(size_t)f * cap + count] = i * nx + j; strength[(size_t)f * cap + count] = row[j]; }
            count++;
          }
        }
      }
      j = p1;
    }
  }
  counts[f] = count;
}

// Fast variant for a compile-time radius: separable window maximum first (row pass, column pass in
// shared memory), so that only pixels equal to their window maximum — a handful per tile — run the
// exact asymmetric predicate.  Same result as nms_bitmask_kernel.
template <int RAD>
__global__ void __launch_bounds__(NMS_NT)
nms_bitmask_sep_kernel(const float *__restrict__ R, unsigned *__restrict__ mask, int nx, int ny, int words_per_row, float Th) {
  constexpr int PW = NMS_TW + 2 * RAD, P = (PW + 3) & ~3, TH2 = NMS_TH + 2 * RAD;   // pitch multiple of 4: 16-byte row loads
  __shared__ __align__(16) float tile[TH2 * P];

  __shared__ __align__(16) float rmax[TH2 * NMS_TW];
  const int x0 = blockIdx.x * NMS_TW, y0 = blockIdx.y * NMS_TH;
  const float *Rf = R + (size_t)nx * ny * blockIdx.z;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  {   // tile rows are streamed by warps; the loads of several rows are issued before the stores
    constexpr int NCH = (PW + 31) / 32;                         // column chunks per row (5)
    constexpr int RPW = (TH2 + 7) / 8;                          // rows per warp (4)
    float v[RPW][NCH];
#pragma unroll
    for (int k = 0; k < RPW; k++) {
      const int r = warp + 8 * k, gy = y0 - RAD + r;
      const bool rowok = r < TH2 && gy >= 0 && gy < ny;
      const float *src = Rf + (size_t)(rowok ? gy : 0) * nx;
#pragma unroll
      for (int q = 0; q < NCH; q++) {
        const int c = lane + 32 * q, gx = x0 - RAD + c;
        v[k][q] = (rowok && c < PW && gx >= 0 && gx < nx) ? __ldg(src + gx) : -INFINITY;
      }
    }
#pragma unroll
    for (int k = 0; k < RPW; k++) {
      const int r = warp + 8 * k;
      if (r < TH2) {
#pragma unroll
        for (int q = 0; q < NCH; q++) { const int c = lane + 32 * q; if (c < PW) tile[r * P + c] = v[k][q]; }
      }
    }
  }
  __syncthreads();
  // row pass: 4 consecutive outputs per item share the middle of their windows
  for (int it = threadIdx.x; it < TH2 * (NMS_TW / 4); it += NMS_NT) {
    const int r = it / (NMS_TW / 4), g = it - r * (NMS_TW / 4);
    const float *p = tile + r * P + 4 * g;                      // output col j covers tile cols j .. j+2*RAD
    constexpr int NV = (4 + 2 * RAD + 3) & ~3;
    float v[NV];
#pragma unroll
    for (int q = 0; q < NV / 4; q++) {
      const float4 t = *reinterpret_cast<const float4 *>(p + 4 * q);
      v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
    float mid = v[3];
#pragma unroll
    for (int q = 4; q <= 2 * RAD; q++) mid = fmaxf(mid, v[q]);  // cols 3 .. 2*RAD are in all four windows
    float o0 = fmaxf(fmaxf(mid, v[0]), fmaxf(v[1], v[2]));
    float o1 = fmaxf(fmaxf(mid, v[1]), fmaxf(v[2], v[2 * RAD + 1]));
    float o2 = fmaxf(fmaxf(mid, v[2]), fmaxf(v[2 * RAD + 1], v[2 * RAD + 2]));
    float o3 = fmaxf(fmaxf(mid, v[2 * RAD + 1]), fmaxf(v[2 * RAD + 2], v[2 * RAD + 3]));
    *reinterpret_cast<float4 *>(rmax + r * NMS_TW + 4 * g) = make_float4(o0, o1, o2, o3);
  }
  __syncthreads();
  // column pass + candidate test: thread = (column, group of 8 rows); lanes of a warp = 32 consecutive columns
  {
    const int col = threadIdx.x & (NMS_TW - 1), rg = threadIdx.x / NMS_TW;       // 2 row groups
    float v[8 + 2 * RAD];
#pragma unroll
    for (int q = 0; q < 8 + 2 * RAD; q++) v[q] = rmax[(rg * 8 + q) * NMS_TW + col];
#pragma unroll
    for (int j = 0; j < 8; j++) {
      float m = v[j];
#pragma unroll
      for (int q = 1; q <= 2 * RAD; q++) m = fmaxf(m, v[j + q]);
      const int row = rg * 8 + j, gx = x0 + col, gy = y0 + row;
      const float *c = tile + (row + RAD) * P + col + RAD;
      const float val = *c;
      bool ok = gx >= RAD && gx < nx - RAD && gy >= RAD && gy < ny - RAD && !(val < Th) && val >= m;
      if (ok && gx == RAD && c[-1] >= val) ok = false;   // harris.cpp:173
      if (ok) {       // val equals its window maximum: apply the reference's tie rules exactly
        for (int dy = -RAD; dy <= RAD && ok; dy++) {
          const float *q = c + dy * P;
          if (dy < 0) { for (int dx = -RAD; dx <= RAD; dx++) ok = ok && (val > q[dx]); }
          else if (dy > 0) { for (int dx = -RAD; dx <= RAD; dx++) ok = ok && (val >= q[dx]); }
          else {
            for (int dx = -RAD; dx < 0; dx++) ok = ok && (val >= q[dx]);
            for (int dx = 1; dx <= RAD; dx++) ok = ok && (val > q[dx]);
          }
        }
      }
      const unsigned bits = __ballot_sync(0xffffffffu, ok);
      const int word = (x0 >> 5) + (col >> 5);
      if (lane == 0 && gy < ny && word < words_per_row) mask[((size_t)blockIdx.z * ny + gy) * words_per_row + word] = bits;
    }
  }
}

// one warp per row: number of set bits of that row
__global__ void row_count_kernel(const unsigned *__restrict__ mask, int *__restrict__ row_cnt, int ny, int words_per_row) {
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31, f = blockIdx.y;
  if (row >= ny) return;
  const unsigned *m = mask + ((size_t)f * ny + row) * words_per_row;
  int c = 0;
  for (int w = lane; w < words_per_row; w += 32) c += __popc(m[w]);
  for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if (lane == 0) row_cnt[(size_t)f * ny + row] = c;
}
// per frame (one CTA): exclusive scan of the row counts, in place; total -> counts[f]
__global__ void __launch_bounds__(1024)
row_scan_kernel(int *__restrict__ row_off, int *__restrict__ counts, int ny) {
  __shared__ int warp_tot[32];
  __shared__ int carry;
  int *off = row_off + (size_t)blockIdx.x * ny;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < ny; base += blockDim.x) {
    int row = base + threadIdx.x;
    int mycount = row < ny ? off[row] : 0;
    int incl = mycount;
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int t = lane < nwarp ? warp_tot[lane] : 0;
      int ti = t;
      for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
      warp_tot[lane] = ti - t;   // exclusive
    }
    __syncthreads();
    int excl = carry + warp_tot[warp] + incl - mycount;
    if (row < ny) off[row] = excl;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry = excl + mycount;
    __syncthreads();
  }
  if (threadIdx.x == 0) counts[blockIdx.x] = carry;
}

// one warp per row: expand the bitmask into (y*nx+x, R) records at the scanned offsets
__global__ void emit_corners_kernel(const unsigned *__restrict__ mask, const int *__restrict__ row_off,
                                    const float *__restrict__ R, int *__restrict__ xy, float *__restrict__ strength,
                                    int nx, int ny, int words_per_row, int cap) {
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31, f = blockIdx.y;
  if (row >= ny) return;
  const unsigned *m = mask + ((size_t)f * ny + row) * words_per_row;
  int base = row_off[(size_t)f * ny + row];
  for (int w0 = 0; w0 < words_per_row; w0 += 32) {
    int w = w0 + lane;
    unsigned bits = w < words_per_row ? m[w] : 0u;
    int c = __popc(bits), incl = c;
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    int pos = base + incl - c;
    while (bits) {
      int b = __ffs(bits) - 1;
      bits &= bits - 1;
      int x = w * 32 + b;
      if (pos < cap) {
        xy[(size_t)f * cap + pos] = row * nx + x;
        strength[(size_t)f * cap + pos] = R[((size_t)f * ny + row) * nx + x];
      }
      pos++;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// gather the 3x3 neighbourhood of selected corners (input of compute_subpixel_precision, harris.cpp:360-369)
__global__ void gather3x3_kernel(const float *__restrict__ R, const int *__restrict__ xy, float *__restrict__ M,
                                 int n, int nx) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int p = xy[i];
  int k = 0;
  for (int dy = -1; dy <= 1; dy++)
    for (int dx = -1; dx <= 1; dx++) M[(size_t)i * 9 + k++] = R[(long long)p + (long long)dy * nx + dx];
}

// Second generation of the separable pre-filter (the first one is issue-bound at ~100 instructions per pixel):
//   * tile 128 x 32 (vertical halo overhead 1.3x instead of 1.6x), columns padded to x0-8 .. x0+135 so that
//     every row is 36 aligned float4 -- six 16-byte loads per thread, no per-element bounds logic inside the image;
//   * both passes use the shared-window trick: G adjacent windows share their middle, the rest are short
//     suffix / prefix maxima -> ~3 max operations per output instead of 2*RAD.
// Candidate rule and exact tie rules are those of nms_bitmask_sep_kernel.
constexpr int NMS2_TW = 128, NMS2_TH = 32, NMS2_LP = 8, NMS2_P = NMS2_TW + 2 * NMS2_LP;

template <int RAD, int G, int B>
__device__ __forceinline__ void window_max_group(const float (&v)[NMS2_TH / 2 + 2 * RAD], float (&out)[NMS2_TH / 2]) {
  // outputs B .. B+G-1: window of output j is v[j .. j+2*RAD]
  float common = v[B + G - 1];
#pragma unroll
  for (int q = B + G; q <= B + 2 * RAD; q++) common = fmaxf(common, v[q]);
  float suf[G], pre[G];
  suf[G - 1] = -INFINITY;
#pragma unroll
  for (int j = G - 2; j >= 0; j--) suf[j] = fmaxf(v[B + j], suf[j + 1]);
  pre[0] = -INFINITY;
#pragma unroll
  for (int j = 1; j < G; j++) pre[j] = fmaxf(pre[j - 1], v[B + 2 * RAD + j]);
#pragma unroll
  for (int j = 0; j < G; j++) out[B + j] = fmaxf(common, fmaxf(suf[j], pre[j]));
}

template <int RAD>
__global__ void __launch_bounds__(NMS_NT)
nms_bitmask_sep2_kernel(const float *__restrict__ R, unsigned *__restrict__ mask, int nx, int ny, int words_per_row, float Th) {
  static_assert(RAD >= 3 && RAD <= NMS2_LP, "radius range of the padded tile");
  constexpr int TH2 = NMS2_TH + 2 * RAD, P = NMS2_P;
  __shared__ __align__(16) float tile[TH2 * P];
  __shared__ __align__(16) float rmax[TH2 * NMS2_TW];
  const int x0 = blockIdx.x * NMS2_TW, y0 = blockIdx.y * NMS2_TH;
  const float *Rf = R + (size_t)nx * ny * blockIdx.z;
  const int lane = threadIdx.x & 31;
  float tmax = -INFINITY;
  if ((nx & 3) == 0 && x0 >= NMS2_LP && x0 + NMS2_TW + NMS2_LP <= nx && y0 >= RAD && y0 + NMS2_TH + RAD <= ny) {
    constexpr int NV4 = TH2 * (P / 4), PER = (NV4 + NMS_NT - 1) / NMS_NT;
    const float *org = Rf + (size_t)(y0 - RAD) * nx + (x0 - NMS2_LP);
    float4 v[PER];
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int u = threadIdx.x + k * NMS_NT, r = u / (P / 4), c4 = u - r * (P / 4);
      v[k] = u < NV4 ? __ldg(reinterpret_cast<const float4 *>(org + (size_t)r * nx + 4 * c4)) : make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    }
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int u = threadIdx.x + k * NMS_NT;
      if (u < NV4) reinterpret_cast<float4 *>(tile)[u] = v[k];
      tmax = fmaxf(tmax, fmaxf(fmaxf(v[k].x, v[k].y), fmaxf(v[k].z, v[k].w)));
    }
  } else {
    for (int u = threadIdx.x; u < TH2 * P; u += NMS_NT) {
      const int r = u / P, c = u - r * P;
      const int gy = y0 - RAD + r, gx = x0 - NMS2_LP + c;
      const float t = (gy >= 0 && gy < ny && gx >= 0 && gx < nx) ? __ldg(Rf + (size_t)gy * nx + gx) : -INFINITY;
      tile[u] = t;
      tmax = fmaxf(tmax, t);
    }
  }
  // A candidate needs R >= Th (harris.cpp:176): a tile none of whose values (halo included) reaches the threshold
  // has an all-zero mask.  On natural frames that is most tiles; the barrier doubles as the vote.  (NaN never votes,
  // and a NaN candidate fails `val >= window max` below as well.)
  if (!__syncthreads_or(!(tmax < Th))) {
    const int row = threadIdx.x >> 2, wq = threadIdx.x & 3;      // 32 rows x 4 mask words
    const int gy = y0 + row, word = (x0 >> 5) + wq;
    if (threadIdx.x < NMS2_TH * 4 && gy < ny && word < words_per_row) mask[((size_t)blockIdx.z * ny + gy) * words_per_row + word] = 0u;
    return;
  }
  // row pass: an item = 4 consecutive outputs of one tile row (output col j <-> tile cols j+8-RAD .. j+8+RAD)
  for (int it = threadIdx.x; it < TH2 * (NMS2_TW / 4); it += NMS_NT) {
    const int r = it >> 5, g = it & 31;
    const float4 *p = reinterpret_cast<const float4 *>(tile + r * P + 4 * g);
    float v[20];
#pragma unroll
    for (int q = 0; q < 5; q++) { const float4 t = p[q]; v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
    constexpr int O = NMS2_LP - RAD;
    float common = v[O + 3];
#pragma unroll
    for (int q = O + 4; q <= O + 2 * RAD; q++) common = fmaxf(common, v[q]);
    const float s2 = v[O + 2], s1 = fmaxf(v[O + 1], s2), s0 = fmaxf(v[O], s1);
    const float p1 = v[O + 2 * RAD + 1], p2 = fmaxf(p1, v[O + 2 * RAD + 2]), p3 = fmaxf(p2, v[O + 2 * RAD + 3]);
    reinterpret_cast<float4 *>(rmax + r * NMS2_TW)[g] =
        make_float4(fmaxf(common, s0), fmaxf(common, fmaxf(s1, p1)), fmaxf(common, fmaxf(s2, p2)), fmaxf(common, p3));
  }
  __syncthreads();
  // column pass + candidate test: thread = (column, half of the tile rows); a warp = 32 consecutive columns = one mask word
  {
    const int col = threadIdx.x & (NMS2_TW - 1), rg = threadIdx.x >> 7;
    constexpr int NR = NMS2_TH / 2;                              // 16 output rows per thread
    float v[NR + 2 * RAD], m[NR];
#pragma unroll
    for (int q = 0; q < NR + 2 * RAD; q++) v[q] = rmax[(rg * NR + q) * NMS2_TW + col];
    constexpr int G = RAD >= 4 ? 8 : 4;
    if (G == 8) { window_max_group<RAD, G, 0>(v, m); window_max_group<RAD, G, 8>(v, m); }
    else { window_max_group<RAD, 4, 0>(v, m); window_max_group<RAD, 4, 4>(v, m); window_max_group<RAD, 4, 8>(v, m); window_max_group<RAD, 4, 12>(v, m); }
    const int gx = x0 + col;
    const bool colok = gx >= RAD && gx < nx - RAD;
    const int word = (x0 >> 5) + (col >> 5);
    const float *c0 = tile + (rg * NR + RAD) * P + col + NMS2_LP;
#pragma unroll
    for (int j = 0; j < NR; j++) {
      const int gy = y0 + rg * NR + j;
      const float *c = c0 + j * P;
      const float val = *c;
      bool ok = colok && gy >= RAD && gy < ny - RAD && !(val < Th) && val >= m[j];
      if (ok && gx == RAD && c[-1] >= val) ok = false;   // harris.cpp:173
      if (ok) {       // val equals its window maximum: apply the reference's tie rules exactly
        for (int dy = -RAD; dy <= RAD && ok; dy++) {
          const float *q = c + dy * P;
          if (dy < 0) { for (int dx = -RAD; dx <= RAD; dx++) ok = ok && (val > q[dx]); }
          else if (dy > 0) { for (int dx = -RAD; dx <= RAD; dx++) ok = ok && (val >= q[dx]); }
          else {
            for (int dx = -RAD; dx < 0; dx++) ok = ok && (val >= q[dx]);
            for (int dx = 1; dx <= RAD; dx++) ok = ok && (val > q[dx]);
          }
        }
      }
      const unsigned bits = __ballot_sync(0xffffffffu, ok);
      if (lane == 0 && gy < ny && word < words_per_row) mask[((size_t)blockIdx.z * ny + gy) * words_per_row + word] = bits;
    }
  }
}

// ------------------------------------------------------------------------------------------
// certified key points on the fast path
//   The fused kernel's R is fp32-accumulated; with it comes, per 8x8 block, a bound eps >= |R - R_ref|
//   (harris_eps).  nms_tolerant_kernel keeps every pixel that COULD satisfy the reference's predicate
//   (harris.cpp:161-243) for some R_ref within the bounds, and marks those for which it certainly does.
//   harris_exact_patch_kernel then repeats the reference's arithmetic (double accumulation in its order,
//   gaussian.cpp:353-358; float products; float measure) on a patch around each candidate: a 1x1 / 3x3 patch
//   for certain ones (their strength, and the 3x3 of the sub-pixel fit), the whole (2r+1)^2 window for the
//   undecided ones, whose predicate is then evaluated on exact values.  compact_kept_kernel keeps the raster order.
// ------------------------------------------------------------------------------------------
constexpr int TN_TW = 128, TN_TH = 32, TN_LP = 8, TN_P = TN_TW + 2 * TN_LP, TN_NT = 256;
constexpr int TN_EBW = TN_P / 8 + 1, TN_EBH = (TN_TH + 2 * 5) / 8 + 2;    // eps blocks a tile (+halo) can touch

template <int RAD>
__global__ void __launch_bounds__(TN_NT)
nms_tolerant_kernel(const float *__restrict__ R, const unsigned *__restrict__ eps_blk, unsigned *__restrict__ cand,
                    unsigned *__restrict__ cert, int nx, int ny, int words_per_row, float Th) {
  static_assert(RAD >= 1 && RAD <= 5, "radius range of the padded tile");
  constexpr int TH2 = TN_TH + 2 * RAD, P = TN_P;
  __shared__ __align__(16) float tile[TH2 * P];                 // L = R - eps rounded down (lower bound of R_ref); -inf outside
  __shared__ __align__(16) float rmax[TH2 * TN_TW];
  __shared__ float epsb[TN_EBH * TN_EBW];
  const int x0 = blockIdx.x * TN_TW, y0 = blockIdx.y * TN_TH;
  const int ebx = (nx + 7) >> 3, eby = (ny + 7) >> 3;
  const float *Rf = R + (size_t)nx * ny * blockIdx.z;
  const float *Ef = reinterpret_cast<const float *>(eps_blk) + (size_t)ebx * eby * blockIdx.z;
  const int bx0 = max(x0 - TN_LP, 0) >> 3, by0 = max(y0 - RAD, 0) >> 3;
  for (int u = threadIdx.x; u < TN_EBH * TN_EBW; u += TN_NT) {
    const int br = u / TN_EBW, bc = u - br * TN_EBW;
    epsb[u] = (by0 + br < eby && bx0 + bc < ebx) ? Ef[(size_t)(by0 + br) * ebx + bx0 + bc] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  float umax = -INFINITY;                                      // largest upper bound in the tile
  if ((nx & 3) == 0 && x0 >= TN_LP && x0 + TN_TW + TN_LP <= nx && y0 >= RAD && y0 + TN_TH + RAD <= ny) {
    // interior tile: 16-byte loads, all of a thread's loads before its stores; the 4 pixels of a vector share an eps block
    constexpr int NV4 = TH2 * (P / 4), PER = (NV4 + TN_NT - 1) / TN_NT;
    const float *org = Rf + (size_t)(y0 - RAD) * nx + (x0 - TN_LP);
    float4 v[PER];
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int u = min((int)threadIdx.x + k * TN_NT, NV4 - 1), r = u / (P / 4), c4 = u - r * (P / 4);
      v[k] = __ldg(reinterpret_cast<const float4 *>(org + (size_t)r * nx + 4 * c4));
    }
#pragma unroll
    for (int k = 0; k < PER; k++) {
      const int u = threadIdx.x + k * TN_NT;
      if (u < NV4) {
        const int r = u / (P / 4), c4 = u - r * (P / 4);
        const float e = epsb[(((y0 - RAD + r) >> 3) - by0) * TN_EBW + (((x0 - TN_LP + 4 * c4) >> 3) - bx0)];
        reinterpret_cast<float4 *>(tile)[u] = make_float4(__fsub_rd(v[k].x, e), __fsub_rd(v[k].y, e), __fsub_rd(v[k].z, e), __fsub_rd(v[k].w, e));
        umax = fmaxf(umax, __fadd_ru(fmaxf(fmaxf(v[k].x, v[k].y), fmaxf(v[k].z, v[k].w)), e));
      }
    }
  } else {
    for (int u = threadIdx.x; u < TH2 * P; u += TN_NT) {
      const int r = u / P, c = u - r * P;
      const int gy = y0 - RAD + r, gx = x0 - TN_LP + c;
      float L = -INFINITY;
      if (gy >= 0 && gy < ny && gx >= 0 && gx < nx) {
        const float v = __ldg(Rf + (size_t)gy * nx + gx);
        const float e = epsb[((gy >> 3) - by0) * TN_EBW + ((gx >> 3) - bx0)];
        L = __fsub_rd(v, e);
        umax = fmaxf(umax, __fadd_ru(v, e));
      }
      tile[u] = L;
    }
  }
  // A corner needs R_ref >= Th: a tile none of whose upper bounds reaches the threshold has empty masks.
  if (!__syncthreads_or(!(umax < Th))) {
    const int row = threadIdx.x >> 2, wq = threadIdx.x & 3;      // 32 rows x 4 mask words
    const int gy = y0 + row, word = (x0 >> 5) + wq;
    if (threadIdx.x < TN_TH * 4 && gy < ny && word < words_per_row) {
      const size_t o = ((size_t)blockIdx.z * ny + gy) * words_per_row + word;
      cand[o] = 0u; cert[o] = 0u;
    }
    return;
  }
  // row pass of the separable window maximum of L
  for (int it = threadIdx.x; it < TH2 * (TN_TW / 4); it += TN_NT) {
    const int r = it >> 5, g = it & 31;
    const float4 *p = reinterpret_cast<const float4 *>(tile + r * P + 4 * g);
    float v[20];
#pragma unroll
    for (int q = 0; q < 5; q++) { const float4 t = p[q]; v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w; }
    constexpr int O = TN_LP - RAD;
    float o[4];
#pragma unroll
    for (int j = 0; j < 4; j++) {
      float m = v[O + j];
#pragma unroll
      for (int q = 1; q <= 2 * RAD; q++) m = fmaxf(m, v[O + j + q]);
      o[j] = m;
    }
    reinterpret_cast<float4 *>(rmax + r * TN_TW)[g] = make_float4(o[0], o[1], o[2], o[3]);
  }
  __syncthreads();
  // column pass + classification: thread = (column, half of the tile rows); a warp = 32 consecutive columns = one mask word
  {
    const int col = threadIdx.x & (TN_TW - 1), rg = threadIdx.x >> 7;
    constexpr int NR = TN_TH / 2;
    const int gx = x0 + col;
    const bool colok = gx >= RAD && gx < nx - RAD;
    const int word = (x0 >> 5) + (col >> 5);
    float win[2 * RAD + 1];
#pragma unroll
    for (int q = 0; q < 2 * RAD; q++) win[q + 1] = rmax[(rg * NR + q) * TN_TW + col];
#pragma unroll 1
    for (int j = 0; j < NR; j++) {
#pragma unroll
      for (int q = 0; q < 2 * RAD; q++) win[q] = win[q + 1];
      win[2 * RAD] = rmax[(rg * NR + j + 2 * RAD) * TN_TW + col];
      float m = win[0];
#pragma unroll
      for (int q = 1; q <= 2 * RAD; q++) m = fmaxf(m, win[q]);
      const int gy = y0 + rg * NR + j;
      bool is_cand = false, is_cert = false;
      if (colok && gy >= RAD && gy < ny - RAD) {
        const float e = epsb[((gy >> 3) - by0) * TN_EBW + ((gx >> 3) - bx0)];
        const float Lp = tile[(rg * NR + j + RAD) * P + col + TN_LP];
        const float Up = fmaf(2.5f, e, Lp);                    // >= R + eps (eps >= 4 ulp(R): harris_eps carries R's own rounding)
        if (Up >= Th && Up >= m) {
          // rare: decide precisely on the window, in double (sums of two floats are exact there)
          const double rp = (double)Rf[(size_t)gy * nx + gx];
          const double up = rp + (double)e, lp = rp - (double)e;
          is_cand = up >= (double)Th;
          is_cert = lp >= (double)Th;
          for (int dy = -RAD; dy <= RAD && is_cand; dy++)
            for (int dx = -RAD; dx <= RAD; dx++) {
              if (dx == 0 && dy == 0) continue;
              const int qy = gy + dy, qx = gx + dx;
              const double rq = (double)Rf[(size_t)qy * nx + qx];
              const double eq = (double)Ef[(size_t)(qy >> 3) * ebx + (qx >> 3)];
              if (rq - eq > up) { is_cand = false; break; }     // q certainly larger: p cannot be a corner
              if (!(rq + eq < lp)) is_cert = false;            // q could be as large as p: undecided
            }
          is_cert = is_cert && is_cand;
        }
      }
      const unsigned bc = __ballot_sync(0xffffffffu, is_cand), bt = __ballot_sync(0xffffffffu, is_cert);
      if (lane == 0 && gy < ny && word < words_per_row) {
        const size_t o = ((size_t)blockIdx.z * ny + gy) * words_per_row + word;
        cand[o] = bc; cert[o] = bt;
      }
    }
  }
}

// one warp per row: expand the candidate mask into (y*nx+x, certain?) records at the scanned offsets
__global__ void emit_candidates_kernel(const unsigned *__restrict__ cand, const unsigned *__restrict__ cert,
                                       const int *__restrict__ row_off, int *__restrict__ xy, unsigned char *__restrict__ flag,
                                       int nx, int ny, int words_per_row, int cap) {
  int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int lane = threadIdx.x & 31, f = blockIdx.y;
  if (row >= ny) return;
  const unsigned *m = cand + ((size_t)f * ny + row) * words_per_row;
  const unsigned *mc = cert + ((size_t)f * ny + row) * words_per_row;
  int base = row_off[(size_t)f * ny + row];
  for (int w0 = 0; w0 < words_per_row; w0 += 32) {
    int w = w0 + lane;
    unsigned bits = w < words_per_row ? m[w] : 0u;
    unsigned cbits = w < words_per_row ? mc[w] : 0u;
    int c = __popc(bits), incl = c;
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    int pos = base + incl - c;
    while (bits) {
      int b = __ffs(bits) - 1;
      bits &= bits - 1;
      if (pos < cap) {
        xy[(size_t)f * cap + pos] = row * nx + w * 32 + b;
        flag[(size_t)f * cap + pos] = (cbits >> b) & 1u;
      }
      pos++;
    }
    base += __shfl_sync(0xffffffffu, incl, 31);
  }
}

// ---- exact patch -------------------------------------------------------------------------------
// Dimensions for the largest case (window radius 5, sigma_i taps 8, sigma_d taps 4).
constexpr int XP_NT = 128;
constexpr int XP_MAXM = 5, XP_MAXRI = 7, XP_MAXRD = 3;
constexpr int XP_PW = 2 * XP_MAXM + 1 + 2 * XP_MAXRI;          // 25 virtual product positions per axis
constexpr int XP_ISW = XP_PW + 2, XP_INW = XP_ISW + 2 * XP_MAXRD;   // 27, 33

struct PatchStats { unsigned long long candidates, undecided, violations, kept; };

template <bool U8>
__global__ void __launch_bounds__(XP_NT)
harris_exact_patch_kernel(const void *__restrict__ frames, const float *__restrict__ Rfused, const unsigned *__restrict__ eps_blk,
                          const int *__restrict__ cand_xy, const unsigned char *__restrict__ cand_flag,
                          const int *__restrict__ cand_cnt, int cap, float *__restrict__ strength, unsigned char *__restrict__ keep,
                          float *__restrict__ M9, PatchStats *__restrict__ stats, int nx, int ny,
                          const __grid_constant__ ExactTaps td, const __grid_constant__ ExactTaps ti,
                          float k, int measure, int grad, float Th, int radius) {
  __shared__ float sI[XP_INW * XP_INW], sT[XP_INW * XP_ISW], sIs[XP_ISW * XP_ISW];
  __shared__ float sP[3][XP_PW * XP_PW], sA[3][XP_PW * (2 * XP_MAXM + 1)], sO[(2 * XP_MAXM + 1) * (2 * XP_MAXM + 1)];
  const int f = blockIdx.y, tid = threadIdx.x;
  const int n = min(cand_cnt[f], cap);
  const int RD = td.size - 1, RI = ti.size - 1;
  const size_t plane = (size_t)nx * ny;
  for (int ci = blockIdx.x; ci < n; ci += gridDim.x) {
    const int p = cand_xy[(size_t)f * cap + ci];
    const bool certain = cand_flag[(size_t)f * cap + ci] != 0;
    const int x = p % nx, y = p / nx;
    // exact R on the (2m+1)^2 patch around (x, y) -> sO (all threads; ends with a barrier)
    auto exact_patch = [&](const int m) {
    const int W = 2 * m + 1, PW = W + 2 * RI;
    // real coordinate ranges (every reflected / replicated coordinate falls inside them, see DESIGN.md)
    const int ix0 = max(0, x - m - RI - 1), ix1 = min(nx - 1, x + m + RI + 1), isw = ix1 - ix0 + 1;
    const int iy0 = max(0, y - m - RI - 1), iy1 = min(ny - 1, y + m + RI + 1), ish = iy1 - iy0 + 1;
    const int cx0 = max(0, ix0 - RD), cx1 = min(nx - 1, ix1 + RD), inw = cx1 - cx0 + 1;
    const int cy0 = max(0, iy0 - RD), cy1 = min(ny - 1, iy1 + RD), inh = cy1 - cy0 + 1;
    __syncthreads();                                           // previous candidate's buffers are free
    for (int i = tid; i < inh * inw; i += XP_NT) {
      const int r = i / inw, c = i - r * inw;
      const size_t g = (size_t)f * plane + (size_t)(cy0 + r) * nx + cx0 + c;
      sI[i] = U8 ? (float)static_cast<const unsigned char *>(frames)[g] : static_cast<const float *>(frames)[g];
    }
    __syncthreads();
    // row pass of discrete_gaussian at sigma_d (gaussian.cpp:332-361): rows cy0..cy1, columns ix0..ix1
    for (int i = tid; i < inh * isw; i += XP_NT) {
      const int r = i / isw, c = i - r * isw, gx = ix0 + c;
      const float *row = sI + r * inw - cx0;
      double sum = __dmul_rn(td.B[0], (double)row[gx]);
      for (int j = 1; j <= RD; j++)
        sum = __dadd_rn(sum, __dmul_rn(td.B[j], __dadd_rn((double)row[pad_index(gx - j, nx)], (double)row[pad_index(gx + j, nx)])));
      sT[i] = __double2float_rn(sum);
    }
    __syncthreads();
    // column pass (gaussian.cpp:363-392): rows iy0..iy1
    for (int i = tid; i < ish * isw; i += XP_NT) {
      const int r = i / isw, c = i - r * isw, gy = iy0 + r;
      const float *col = sT + c - cy0 * isw;
      double sum = __dmul_rn(td.B[0], (double)col[gy * isw]);
      for (int j = 1; j <= RD; j++)
        sum = __dadd_rn(sum, __dmul_rn(td.B[j], __dadd_rn((double)col[pad_index(gy - j, ny) * isw], (double)col[pad_index(gy + j, ny) * isw])));
      sIs[i] = __double2float_rn(sum);
    }
    __syncthreads();
    // gradient (gradient.cpp:17-128) and products (harris.cpp:57-62) at the virtual positions of the sigma_i blur:
    // reflect padding of the product planes, then the replicate rule of the gradient
    for (int i = tid; i < PW * PW; i += XP_NT) {
      const int r = i / PW, c = i - r * PW;
      const int px = min(max(pad_index(x - m - RI + c, nx), 1), nx - 2), py = min(max(pad_index(y - m - RI + r, ny), 1), ny - 2);
      const float *I = sIs + (py - iy0) * isw + (px - ix0);
      float gx, gy;
      if (grad == 1) {
        float hx = __fsub_rn(I[1], I[-1]);
        float dx = __fsub_rn(__fsub_rn(__fadd_rn(I[-isw + 1], I[isw + 1]), I[-isw - 1]), I[isw - 1]);
        gx = __double2float_rn(__dadd_rn(__dmul_rn(0.25, (double)hx), __dmul_rn(0.125, (double)dx)));
        float hy = __fsub_rn(I[isw], I[-isw]);
        float dy = __fsub_rn(__fsub_rn(__fadd_rn(I[isw + 1], I[isw - 1]), I[-isw + 1]), I[-isw - 1]);
        gy = __double2float_rn(__dadd_rn(__dmul_rn(0.25, (double)hy), __dmul_rn(0.125, (double)dy)));
      } else {
        gx = __fmul_rn(0.5f, __fsub_rn(I[1], I[-1]));
        gy = __fmul_rn(0.5f, __fsub_rn(I[isw], I[-isw]));
      }
      sP[0][i] = __fmul_rn(gx, gx); sP[1][i] = __fmul_rn(gx, gy); sP[2][i] = __fmul_rn(gy, gy);
    }
    __syncthreads();
    // sigma_i row pass on the virtual arrays: all PW rows, the W patch columns
    for (int i = tid; i < 3 * PW * W; i += XP_NT) {
      const int pl = i / (PW * W), rr = i - pl * (PW * W), r = rr / W, c = rr - r * W;
      const float *row = sP[pl] + r * PW + c + RI;
      double sum = __dmul_rn(ti.B[0], (double)row[0]);
      for (int j = 1; j <= RI; j++) sum = __dadd_rn(sum, __dmul_rn(ti.B[j], __dadd_rn((double)row[-j], (double)row[j])));
      sA[pl][r * W + c] = __double2float_rn(sum);
    }
    __syncthreads();
    // sigma_i column pass + corner measure (harris.cpp:100-129)
    for (int i = tid; i < W * W; i += XP_NT) {
      const int r = i / W, c = i - r * W;
      float v[3];
      for (int pl = 0; pl < 3; pl++) {
        const float *col = sA[pl] + (r + RI) * W + c;
        double sum = __dmul_rn(ti.B[0], (double)col[0]);
        for (int j = 1; j <= RI; j++) sum = __dadd_rn(sum, __dmul_rn(ti.B[j], __dadd_rn((double)col[-j * W], (double)col[j * W])));
        v[pl] = __double2float_rn(sum);
      }
      sO[i] = corner_measure(v[0], v[1], v[2], k, measure);
    }
    __syncthreads();
    };
    // certain candidates need their own value (and the 3x3 of the sub-pixel fit); undecided ones first their own exact
    // value — most of them sit beside strong edges, where the bound is wide and the exact response is far below the
    // threshold — and the whole window only if that value passes the threshold
    int m = certain ? (M9 ? 1 : 0) : 0;
    exact_patch(m);
    if (!certain && !(sO[0] < Th)) {
      m = radius;
      exact_patch(m);
    }
    const int W = 2 * m + 1;
    if (tid == 0) {
      const float val = sO[m * W + m];
      bool ok = true;
      if (!certain) {                                          // the reference's predicate on exact values (harris.cpp:161-243)
        ok = !(val < Th);                                      // (m == 0 here means exactly that this test failed)
        for (int dy = -m; dy <= m && ok; dy++)
          for (int dx = -m; dx <= m && ok; dx++) {
            const float q = sO[(m + dy) * W + m + dx];
            if (dy < 0) ok = val > q;
            else if (dy > 0) ok = val >= q;
            else if (dx < 0) ok = val >= q;
            else if (dx > 0) ok = val > q;
          }
        if (ok && m > 0 && x == radius && sO[m * W + m - 1] >= val) ok = false;   // harris.cpp:173
      }
      // harris.cpp:175-176 passes over every pixel of the row, from x = radius on, as long as each one is below the
      // threshold, marked, or not above its left neighbour.  A window maximum is passed over only if its left neighbour
      // ties it exactly, and then whether the scan got there depends on the whole row prefix: such a frame is left to
      // the staged kernels (keep = 2 -> count -1).
      const bool tie_left = ok && !certain && m > 0 && x > radius && sO[m * W + m - 1] == val;
      const size_t o = (size_t)f * cap + ci;
      strength[o] = val;
      keep[o] = tie_left ? 2 : (ok ? 1 : 0);
      if (M9 && m >= 1)
        for (int dy = -1; dy <= 1; dy++)
          for (int dx = -1; dx <= 1; dx++) M9[o * 9 + (dy + 1) * 3 + dx + 1] = sO[(m + dy) * W + m + dx];
      // the bound the decision relied on must hold: counted, and asserted == 0 by the tests
      const float e = reinterpret_cast<const float *>(eps_blk)[((size_t)f * ((ny + 7) >> 3) + (y >> 3)) * ((nx + 7) >> 3) + (x >> 3)];
      const float rf = Rfused[(size_t)f * plane + p];
      if (!(fabs((double)rf - (double)val) <= (double)e)) atomicAdd(&stats->violations, 1ull);
      if (!certain) atomicAdd(&stats->undecided, 1ull);
      if (ok) atomicAdd(&stats->kept, 1ull);
      if (ci == 0) atomicAdd(&stats->candidates, (unsigned long long)n);
    }
  }
}

// one CTA per frame: stable compaction of the kept candidates (raster order of harris.cpp:250-252)
__global__ void __launch_bounds__(1024)
compact_kept_kernel(const int *__restrict__ cand_xy, const unsigned char *__restrict__ keep, const float *__restrict__ cand_s,
                    const float *__restrict__ cand_M9, const int *__restrict__ cand_cnt, int cand_cap,
                    int *__restrict__ xy, float *__restrict__ strength, float *__restrict__ M9, int *__restrict__ counts, int cap) {
  __shared__ int warp_tot[32];
  __shared__ int carry, undecidable;
  const int f = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n = min(cand_cnt[f], cand_cap);
  if (threadIdx.x == 0) { carry = 0; undecidable = 0; }
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int i = base + threadIdx.x;
    const size_t ci = (size_t)f * cand_cap + i;
    const int kflag = (i < n && keep[ci]) ? 1 : 0;
    if (i < n && keep[ci] == 2) undecidable = 1;
    int incl = kflag;
    for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int t = warp_tot[lane], ti = t;
      for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
      warp_tot[lane] = ti - t;
    }
    __syncthreads();
    const int pos = carry + warp_tot[warp] + incl - kflag;
    if (kflag && pos < cap) {
      const size_t o = (size_t)f * cap + pos;
      xy[o] = cand_xy[ci];
      strength[o] = cand_s[ci];
      if (M9) for (int q = 0; q < 9; q++) M9[o * 9 + q] = cand_M9[ci * 9 + q];
    }
    __syncthreads();
    if (threadIdx.x == 1023) carry = pos + kflag;
    __syncthreads();
  }
  // more candidates than record slots (the list is incomplete), or a corner the row scan may pass over: say so (callers
  // rerun the frame through the staged kernels)
  if (threadIdx.x == 0) counts[f] = (cand_cnt[f] > cand_cap || undecidable) ? -1 : carry;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
// exact staged path: d_I (float planes) is blurred IN PLACE like harris.cpp:511, R written to d_R.
// Scratch: 4 float planes per frame (+ SII line buffers) from the arena.
static int response_exact(b2f_ctx *ctx, float *d_I, int n_frames, int nx, int ny, const b2f_harris_params *p,
                          float *d_R, cudaStream_t st) {
  size_t plane = (size_t)nx * ny, tot = plane * n_frames;
  float *T = ctx->arena.get<float>(tot), *A = ctx->arena.get<float>(tot), *B = ctx->arena.get<float>(tot),
        *Cc = ctx->arena.get<float>(tot);
  int g1 = p->gaussian, g2 = (p->gaussian == 2) ? 1 : p->gaussian;   // harris.cpp:64-65
  const int nmax = nx > ny ? nx : ny;
  float *sii_scratch = nullptr;
  if (g1 == 1 || g2 == 1) {
    // largest pad among the two sigmas
    double sg = std::max(p->sigma_d, p->sigma_i);
    int pad = (int)(76 * (sg / (100.0 / 3.14159265358979323846264338327950288)) + 0.5) + 1;
    sii_scratch = ctx->arena.get<float>((size_t)n_frames * nmax * (nmax + 2 * pad));
  }
  B2F_ARENA_CHECK(ctx);

  auto blur = [&](float *buf, float sigma, int type) -> int {   // gaussian(): gaussian.cpp:403-430, in place
    if (type == 0) {
      if (sigma <= 0) return B2F_OK;                               // copy of itself
      ExactTaps tp;
      tp.size = harris_taps_double(sigma, tp.B);
      if (tp.size < 0) { set_error("harris: sigma %.3f needs more than %d taps", sigma, HARRIS_MAX_TAPS); return B2F_EUNSUP; }
      if (tp.size > nx) return B2F_OK;                             // gaussian.cpp:312 early-out
      if (tp.size > ny) { set_error("harris: image height %d below the Gaussian half-width %d (undefined in the reference)", ny, tp.size); return B2F_EUNSUP; }
      dim3 grid(ceil_div(nx, 128), ny, n_frames);
      exact_gauss_pass<false><<<grid, 128, 0, st>>>(buf, T, nx, ny, tp);
      B2F_LAUNCH_CHECK(ctx);
      exact_gauss_pass<true><<<grid, 128, 0, st>>>(T, buf, nx, ny, tp);
      B2F_LAUNCH_CHECK(ctx);
      return B2F_OK;
    }
    if (type == 1) {
      SiiCoef c;                                                   // gaussian.cpp:61-90, K=3
      const double sigma0 = 100.0 / 3.14159265358979323846264338327950288;
      static const short radii0[3] = {76, 46, 23};
      static const float weights0[3] = {0.1618f, 0.5502f, 0.9495f};
      double sum = 0;
      for (int k = 0; k < 3; k++) {
        c.r[k] = (int)(long)(radii0[k] * ((double)sigma / sigma0) + 0.5);
        sum += weights0[k] * (2 * (long)c.r[k] + 1);
      }
      for (int k = 0; k < 3; k++) c.w[k] = (float)(weights0[k] / sum);
      exact_sii_pass<<<dim3(ceil_div(ny, 64), n_frames), 64, 0, st>>>(buf, T, sii_scratch, nx, ny, 0, c);
      B2F_LAUNCH_CHECK(ctx);
      exact_sii_pass<<<dim3(ceil_div(nx, 64), n_frames), 64, 0, st>>>(T, buf, sii_scratch, nx, ny, 1, c);
      B2F_LAUNCH_CHECK(ctx);
      return B2F_OK;
    }
    return B2F_OK;   // NO_GAUSSIAN: copy of itself
  };
  int rc;
  if ((rc = blur(d_I, p->sigma_d, g1)) != B2F_OK) return rc;
  dim3 grid(ceil_div(nx, 128), ny, n_frames);
  exact_grad_products<<<grid, 128, 0, st>>>(d_I, A, B, Cc, nx, ny, p->gradient == 1 ? 1 : 0);
  B2F_LAUNCH_CHECK(ctx);
  if ((rc = blur(A, p->sigma_i, g2)) != B2F_OK) return rc;
  if ((rc = blur(B, p->sigma_i, g2)) != B2F_OK) return rc;
  if ((rc = blur(Cc, p->sigma_i, g2)) != B2F_OK) return rc;
  exact_response<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(A, B, Cc, d_R, tot, p->k, p->measure);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

// response map for frames already on the device.  exact!=0 forces the staged bit-exact path.
// For the exact path with u8 input (or when the caller's float planes must stay untouched) the
// frames are first copied into arena scratch.
int harris_response_device(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny,
                           const b2f_harris_params *p, int exact, float *d_R, cudaStream_t st) {
  if (!exact && harris_fused_supported(nx, ny, p->sigma_d, p->sigma_i, p->gaussian))
    return harris_fused_launch(ctx, d_frames, u8, n_frames, nx, ny, p, d_R, nullptr, false, st);
  size_t tot = (size_t)nx * ny * n_frames;
  float *I = ctx->arena.get<float>(tot);
  B2F_ARENA_CHECK(ctx);
  if (u8) {
    u8_to_float<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(static_cast<const unsigned char *>(d_frames), I, tot);
    B2F_LAUNCH_CHECK(ctx);
  } else {
    B2F_CUDA(cudaMemcpyAsync(I, d_frames, tot * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return response_exact(ctx, I, n_frames, nx, ny, p, d_R, st);
}

int harris_nms_device(b2f_ctx *ctx, const float *d_R, int n_frames, int nx, int ny, float Th, int radius, int cap,
                      int *d_xy, float *d_strength, int *d_counts, cudaStream_t st) {
  if (radius < 1) radius = 1;                                   // harris.cpp:152 (after the size check :151)
  const int wpr = ceil_div(nx, 32);
  unsigned *mask = ctx->arena.get<unsigned>((size_t)n_frames * ny * wpr);
  int *row_off = ctx->arena.get<int>((size_t)n_frames * ny);
  unsigned char *skip = ctx->arena.get<unsigned char>((size_t)n_frames * nx * ny);
  B2F_ARENA_CHECK(ctx);
  size_t smem = sizeof(float) * (size_t)(NMS_TW + 2 * radius) * (NMS_TH + 2 * radius);
  if (smem > 200 * 1024) { set_error("harris: NMS radius %d too large", radius); return B2F_EUNSUP; }
  if (smem > 48 * 1024) B2F_CUDA(cudaFuncSetAttribute(nms_bitmask_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  dim3 grid(ceil_div(nx, NMS_TW), ceil_div(ny, NMS_TH), n_frames);
  static const bool sep1 = getenv("B2F_NMS_SEP1") != nullptr;
  dim3 grid2(ceil_div(nx, NMS2_TW), ceil_div(ny, NMS2_TH), n_frames);
  if (radius == 5 && !sep1) nms_bitmask_sep2_kernel<5><<<grid2, NMS_NT, 0, st>>>(d_R, mask, nx, ny, wpr, Th);
  else if (radius == 3 && !sep1) nms_bitmask_sep2_kernel<3><<<grid2, NMS_NT, 0, st>>>(d_R, mask, nx, ny, wpr, Th);
  else if (radius == 5) nms_bitmask_sep_kernel<5><<<grid, NMS_NT, 0, st>>>(d_R, mask, nx, ny, wpr, Th);
  else if (radius == 3) nms_bitmask_sep_kernel<3><<<grid, NMS_NT, 0, st>>>(d_R, mask, nx, ny, wpr, Th);
  else nms_bitmask_kernel<<<grid, NMS_NT, smem, st>>>(d_R, mask, nx, ny, wpr, Th, radius);
  B2F_LAUNCH_CHECK(ctx);
  row_count_kernel<<<dim3(ceil_div(ny, 8), n_frames), 256, 0, st>>>(mask, row_off, ny, wpr);
  B2F_LAUNCH_CHECK(ctx);
  row_scan_kernel<<<n_frames, 1024, 0, st>>>(row_off, d_counts, ny);
  B2F_LAUNCH_CHECK(ctx);
  emit_corners_kernel<<<dim3(ceil_div(ny, 8), n_frames), 256, 0, st>>>(mask, row_off, d_R, d_xy, d_strength, nx, ny, wpr, cap);
  B2F_LAUNCH_CHECK(ctx);
  nms_tie_rescan_kernel<<<n_frames, 256, 0, st>>>(d_R, mask, skip, nx, ny, wpr, Th, radius, cap, d_xy, d_strength, d_counts);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

int mask_row_offsets(b2f_ctx *ctx, const unsigned *mask, int *row_off, int *d_counts, int n_frames, int ny, int wpr, cudaStream_t st) {
  row_count_kernel<<<dim3(ceil_div(ny, 8), n_frames), 256, 0, st>>>(mask, row_off, ny, wpr);
  B2F_LAUNCH_CHECK(ctx);
  row_scan_kernel<<<n_frames, 1024, 0, st>>>(row_off, d_counts, ny);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

// ---- certified corners on the fast path ---------------------------------------------------------
bool harris_certified_supported(int nx, int ny, const b2f_harris_params *p) {
  if (!harris_fused_supported(nx, ny, p->sigma_d, p->sigma_i, p->gaussian)) return false;
  if (p->measure != 0) return false;                            // the error bound is derived for the Harris measure
  const int radius = 2 * p->sigma_i + 0.5;                      // harris.cpp:523
  if (!(radius == 2 || radius == 3 || radius == 5)) return false;
  return !(ny <= 2 * radius + 1 || nx <= 2 * radius + 1);
}

size_t harris_certified_scratch_bytes(int n_frames, int nx, int ny, int cap, bool want_m9) {
  const size_t wpr = ceil_div(nx, 32), ebx = (nx + 7) >> 3, eby = (ny + 7) >> 3;
  size_t b = align256((size_t)n_frames * nx * ny * 4);                          // R
  b += align256((size_t)n_frames * ebx * eby * 4);                               // eps blocks
  b += 2 * align256((size_t)n_frames * ny * wpr * 4) + align256((size_t)n_frames * ny * 4);   // masks, row offsets
  b += align256((size_t)n_frames * cap * 4) * 2 + align256((size_t)n_frames * cap) * 2 + align256((size_t)n_frames * 4);
  if (want_m9) b += align256((size_t)n_frames * cap * 36);
  return b + 4096;
}

// frames (u8 or float, resident on the device) -> raster-ordered corner lists identical to the reference's:
// d_xy[f*cap + i] = y*nx + x, d_strength = the reference's R there (bit for bit), d_M9 (optional) its 3x3
// neighbourhood, d_counts[f] = number of corners (may exceed cap: the caller reports B2F_ECAP).
// d_R_out (optional) receives the fp32 response planes.  Scratch from the arena (harris_certified_scratch_bytes).
int harris_corners_certified(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny,
                             const b2f_harris_params *p, int cap, int *d_xy, float *d_strength, float *d_M9,
                             int *d_counts, float *d_R_out, cudaStream_t st) {
  const int radius = 2 * p->sigma_i + 0.5;
  const size_t plane = (size_t)nx * ny;
  const int wpr = ceil_div(nx, 32), ebx = (nx + 7) >> 3, eby = (ny + 7) >> 3;
  float *d_R = d_R_out ? d_R_out : ctx->arena.get<float>(plane * n_frames);
  unsigned *eps = ctx->arena.get<unsigned>((size_t)n_frames * ebx * eby);
  unsigned *cand = ctx->arena.get<unsigned>((size_t)n_frames * ny * wpr);
  unsigned *cert = ctx->arena.get<unsigned>((size_t)n_frames * ny * wpr);
  int *row_off = ctx->arena.get<int>((size_t)n_frames * ny);
  int *c_xy = ctx->arena.get<int>((size_t)n_frames * cap);
  float *c_s = ctx->arena.get<float>((size_t)n_frames * cap);
  unsigned char *c_flag = ctx->arena.get<unsigned char>((size_t)n_frames * cap);
  unsigned char *c_keep = ctx->arena.get<unsigned char>((size_t)n_frames * cap);
  int *c_cnt = ctx->arena.get<int>(n_frames);
  float *c_M9 = d_M9 ? ctx->arena.get<float>((size_t)n_frames * cap * 9) : nullptr;
  B2F_ARENA_CHECK(ctx);
  if (!ctx->harris_stats) {
    B2F_CUDA(cudaMalloc(&ctx->harris_stats, sizeof(PatchStats)));
    B2F_CUDA(cudaMemsetAsync(ctx->harris_stats, 0, sizeof(PatchStats), st));
  }
  B2F_CUDA(cudaMemsetAsync(eps, 0, sizeof(unsigned) * (size_t)n_frames * ebx * eby, st));
  int rc = harris_fused_launch(ctx, d_frames, u8, n_frames, nx, ny, p, d_R, eps, true, st);
  if (rc != B2F_OK) return rc;
  dim3 grid(ceil_div(nx, TN_TW), ceil_div(ny, TN_TH), n_frames);
  if (radius == 5) nms_tolerant_kernel<5><<<grid, TN_NT, 0, st>>>(d_R, eps, cand, cert, nx, ny, wpr, p->threshold);
  else if (radius == 3) nms_tolerant_kernel<3><<<grid, TN_NT, 0, st>>>(d_R, eps, cand, cert, nx, ny, wpr, p->threshold);
  else nms_tolerant_kernel<2><<<grid, TN_NT, 0, st>>>(d_R, eps, cand, cert, nx, ny, wpr, p->threshold);
  B2F_LAUNCH_CHECK(ctx);
  row_count_kernel<<<dim3(ceil_div(ny, 8), n_frames), 256, 0, st>>>(cand, row_off, ny, wpr);
  B2F_LAUNCH_CHECK(ctx);
  row_scan_kernel<<<n_frames, 1024, 0, st>>>(row_off, c_cnt, ny);
  B2F_LAUNCH_CHECK(ctx);
  emit_candidates_kernel<<<dim3(ceil_div(ny, 8), n_frames), 256, 0, st>>>(cand, cert, row_off, c_xy, c_flag, nx, ny, wpr, cap);
  B2F_LAUNCH_CHECK(ctx);
  ExactTaps td, ti;
  td.size = harris_taps_double(p->sigma_d, td.B);
  ti.size = harris_taps_double(p->sigma_i, ti.B);
  if (td.size - 1 > XP_MAXRD || ti.size - 1 > XP_MAXRI || radius > XP_MAXM) { set_error("harris: patch dimensions exceeded"); return B2F_EUNSUP; }
  PatchStats *stats = static_cast<PatchStats *>(ctx->harris_stats);
  const dim3 pgrid(std::max(1, std::min(cap, 2 * ctx->sm_count)), n_frames);
  if (u8) harris_exact_patch_kernel<true><<<pgrid, XP_NT, 0, st>>>(d_frames, d_R, eps, c_xy, c_flag, c_cnt, cap, c_s, c_keep, c_M9, stats, nx, ny,
                                                                   td, ti, p->k, p->measure, p->gradient == 1 ? 1 : 0, p->threshold, radius);
  else harris_exact_patch_kernel<false><<<pgrid, XP_NT, 0, st>>>(d_frames, d_R, eps, c_xy, c_flag, c_cnt, cap, c_s, c_keep, c_M9, stats, nx, ny,
                                                                  td, ti, p->k, p->measure, p->gradient == 1 ? 1 : 0, p->threshold, radius);
  B2F_LAUNCH_CHECK(ctx);
  compact_kept_kernel<<<n_frames, 1024, 0, st>>>(c_xy, c_keep, c_s, c_M9, c_cnt, cap, d_xy, d_strength, d_M9, d_counts, cap);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

// candidates / undecided / bound violations / kept since the context was created (synchronises `st`)
int harris_cert_stats(b2f_ctx *ctx, unsigned long long out[4], cudaStream_t st) {
  out[0] = out[1] = out[2] = out[3] = 0;
  if (!ctx->harris_stats) return B2F_OK;
  PatchStats h;
  B2F_CUDA(cudaMemcpyAsync(&h, ctx->harris_stats, sizeof(h), cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  out[0] = h.candidates; out[1] = h.undecided; out[2] = h.violations; out[3] = h.kept;
  return B2F_OK;
}

int harris_gather3x3(b2f_ctx *ctx, const float *d_R, const int *d_xy, float *d_M, int n, int nx, cudaStream_t st) {
  if (n <= 0) return B2F_OK;
  gather3x3_kernel<<<ceil_div(n, 256), 256, 0, st>>>(d_R, d_xy, d_M, n, nx);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

int harris_decimate2(b2f_ctx *ctx, const float *d_src, float *d_dst, int nx, int ny, cudaStream_t st) {
  decimate2<<<dim3(ceil_div(nx / 2, 128), ny / 2), 128, 0, st>>>(d_src, d_dst, nx, ny);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

__global__ void double_to_float_kernel(const double *__restrict__ s, float *__restrict__ d, size_t n) {   // I[i] = (float)x[i], rcpp_harris.cpp:35
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) d[i] = __double2float_rn(s[i]);
}
int harris_double_to_float(b2f_ctx *ctx, const double *s, float *d, size_t n, cudaStream_t st) {
  double_to_float_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s, d, n);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

int harris_u8_to_float(b2f_ctx *ctx, const unsigned char *s, float *d, size_t n, cudaStream_t st) {
  u8_to_float<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(s, d, n);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

}  // namespace b2f
