// fhog.cu — Felzenszwalb HOG of dlib 19.20 as reached from image.dlib::image_fhog
// (SURVEY.md §8a rows F1-F2; reference: dlib/image_transforms/fhog.h:698-1046).
//
//   fhog_lut_kernel      (once per context) 511 x 511 table of the 18-way orientation snap for every
//                        possible integer gradient (gx, gy in -255..255), computed with the reference's
//                        un-fused float ops (fhog.h:864-877) -> the per-pixel snap is one table load.
//   fhog_pixel_kernel    one CTA = a 64 x 16 pixel tile (+1 ring, word-aligned staging of the RGB bytes).
//                        Per pixel: max-length colour channel with the reference's position-dependent
//                        tie-break (SIMD body vs scalar tail, fhog.h:48-58 / :133-141), LUT snap,
//                        correctly rounded sqrt.  A thread takes 4 consecutive rows of one column (column-only
//                        work is formed once).  Writes a magnitude plane and an orientation plane in a
//                        cell-phase de-interleaved column order, so the next kernel's loads coalesce.
//   fhog_cell_kernel     ONE thread per histogram cell replays that cell's votes in raster order (the
//                        order of the reference's sequential `hist += v` statements, fhog.h:879-917,
//                        :951-954), accumulating in a private shared-memory histogram -> the 18-bin
//                        histograms are BIT-IDENTICAL to the reference, no atomics.
//   fhog_norm_kernel     per-cell energy (fhog.h:959-968), sequential over the 9 orientations.
//   fhog_feature_kernel  4-block normalisation, clipping and the 31 features (fhog.h:972-1045)
//                        with the SSE2 lane and summation order ((l0+l2)+(l1+l3), simd4f.h:549-566).
// Bilinear weights and cell indices come from per-row / per-column tables built on the host with
// the reference's own float expressions (fhog.h:823-826, :838-841, :946-949).
#include "common.cuh"
#include <cmath>
#include <vector>

namespace b2f {

struct FhogGeom {
  int rows, cols, cell;
  int cells_nr, cells_nc, hog_nr, hog_nc;   // hog_* without padding
  int visible_nr, visible_nc, simd_end;
  int out_nr, out_nc, pad_r, pad_c;
};

static bool fhog_geometry(int rows, int cols, int cell, int frp, int fcp, FhogGeom &g) {
  g.rows = rows; g.cols = cols; g.cell = cell;
  g.cells_nr = (int)((float)rows / (float)cell + 0.5);                      // fhog.h:780-781
  g.cells_nc = (int)((float)cols / (float)cell + 0.5);
  g.hog_nr = std::max(g.cells_nr - 2, 0); g.hog_nc = std::max(g.cells_nc - 2, 0);
  g.out_nr = g.out_nc = 0; g.pad_r = (frp - 1) / 2; g.pad_c = (fcp - 1) / 2;
  if (g.cells_nr == 0 || g.cells_nc == 0 || g.hog_nr == 0 || g.hog_nc == 0) return false;   // hog.clear()
  g.out_nr = g.hog_nr + frp - 1; g.out_nc = g.hog_nc + fcp - 1;             // init_hog, fhog.h:457
  g.visible_nr = (int)std::min((long)g.cells_nr * cell, (long)rows) - 1;    // fhog.h:817-818
  g.visible_nc = (int)std::min((long)g.cells_nc * cell, (long)cols) - 1;
  int x = 1;
  for (; x < g.visible_nc - 7; x += 8) {}
  g.simd_end = x;                                                           // columns < simd_end: simd8 body
  return true;
}

// per-row / per-column vote tables
struct FhogTables {
  const short *r0, *c0;            // first histogram row / column a pixel votes into
  const float *vy0, *vy1, *vx0, *vx1;
  const int *ylo, *yhi, *xlo, *xhi;   // pixel range voting into histogram row R / column C
};

constexpr int FH_NT = 256;

__device__ __forceinline__ void snap18(float gx, float gy, int &best_o) {
  const float DX[9] = {1.0000f, 0.9397f, 0.7660f, 0.500f, 0.1736f, -0.1736f, -0.5000f, -0.7660f, -0.9397f};
  const float DY[9] = {0.0000f, 0.3420f, 0.6428f, 0.8660f, 0.9848f, 0.9848f, 0.8660f, 0.6428f, 0.3420f};
  float best = 0.f;
  best_o = 0;
#pragma unroll
  for (int o = 0; o < 9; o++) {
    float d = __fadd_rn(__fmul_rn(gx, DX[o]), __fmul_rn(gy, DY[o]));
    if (d > best) { best = d; best_o = o; }
    else if (-d > best) { best = -d; best_o = o + 9; }
  }
}

// ---- pass 1: per-pixel (orientation bin, gradient magnitude), written in a cell-phase
// de-interleaved layout  idx(y,x) = y*PW + (x % cell)*NCB + x / cell  so that pass 2 (one thread per
// cell, consecutive threads = consecutive cells) reads consecutive addresses.
constexpr int FC_NT = 128;                                 // threads (= histogram cells) per CTA of the cell kernel
constexpr int FP_TW = 64, FP_TH = 16;
constexpr int FP_RB = ((FP_TW + 2) * 3 + 3 + 15) & ~15;    // staged bytes per row (208): 16-byte chunks, + up to 3 lead bytes

// 18-way orientation snap for every integer gradient (gx, gy) in [-255, 255]^2, built once per
// context with the same un-fused float expressions (snap18): lut[(gy+255)*512 + gx+255].
__global__ void fhog_lut_kernel(unsigned char *__restrict__ lut) {
  int gx = (int)(blockIdx.x * blockDim.x + threadIdx.x) - 255, gy = (int)blockIdx.y - 255;
  if (gx > 255) return;
  int o;
  snap18((float)gx, (float)gy, o);
  lut[(gy + 255) * 512 + gx + 255] = (unsigned char)o;
}

__global__ void __launch_bounds__(FH_NT)
fhog_pixel_kernel(const unsigned char *__restrict__ frames, float *__restrict__ vmag, unsigned char *__restrict__ obin,
                  FhogGeom g, const int *__restrict__ colidx, int PW, const unsigned char *__restrict__ lut, int aligned) {
  __shared__ __align__(16) unsigned char srgb[(FP_TH + 2) * FP_RB];
  const int x0 = 1 + blockIdx.x * FP_TW, y0 = 1 + blockIdx.y * FP_TH;       // voters live in [1, visible)
  const unsigned char *src = frames + (size_t)blockIdx.z * g.rows * g.cols * 3;
  const int b0 = (x0 - 1) * 3;                      // first byte of the staged row segment
  const int lead = aligned ? (b0 & 3) : 0;          // bytes in front of it when loading whole words
  const int rowlimit = g.cols * 3;
  if (aligned == 2) {
    // rows are multiples of 16 bytes and b0 = 192 * blockIdx.x: 13 aligned 16-byte chunks per row, one per thread
    if (threadIdx.x < (FP_TH + 2) * (FP_RB / 16)) {
      const int r = threadIdx.x / (FP_RB / 16), q = threadIdx.x - r * (FP_RB / 16);
      const int gy = min(y0 - 1 + r, g.rows - 1), gb = b0 + 16 * q;
      const unsigned char *row = src + (size_t)gy * rowlimit;
      uint4 v;
      if (gb + 16 <= rowlimit) v = __ldg(reinterpret_cast<const uint4 *>(row + gb));
      else {      // chunk crosses the end of the row: words past it are never read by a voter
        unsigned w[4];
#pragma unroll
        for (int k = 0; k < 4; k++) w[k] = gb + 4 * k + 4 <= rowlimit ? __ldg(reinterpret_cast<const unsigned *>(row + gb + 4 * k)) : 0u;
        v = make_uint4(w[0], w[1], w[2], w[3]);
      }
      reinterpret_cast<uint4 *>(srgb)[r * (FP_RB / 16) + q] = v;
    }
  } else if (aligned) {
    const int w0 = (b0 - lead) >> 2;
    for (int i = threadIdx.x; i < (FP_TH + 2) * (FP_RB / 4); i += FH_NT) {
      int r = i / (FP_RB / 4), w = i - r * (FP_RB / 4);
      int gy = min(y0 - 1 + r, g.rows - 1);
      int wb = min((w0 + w) * 4, rowlimit - 4);     // rows are multiples of 4 bytes on this path
      reinterpret_cast<unsigned *>(srgb)[r * (FP_RB / 4) + w] = __ldg(reinterpret_cast<const unsigned *>(src + (size_t)gy * rowlimit + wb));
    }
  } else {
    for (int i = threadIdx.x; i < (FP_TH + 2) * FP_RB; i += FH_NT) {
      int r = i / FP_RB, b = i - r * FP_RB;
      int gy = min(y0 - 1 + r, g.rows - 1), gxb = min(b0 + b, rowlimit - 1);
      srgb[i] = __ldg(src + (size_t)gy * rowlimit + gxb);
    }
  }
  __syncthreads();
  // thread = (column c, group of 4 consecutive rows): everything that depends on the column alone -- the
  // SIMD-body / scalar-tail rule, the de-interleaved output column, the staged byte offset -- is formed once
  const int c = threadIdx.x & (FP_TW - 1), rg = threadIdx.x >> 6;
  const int x = x0 + c;
  if (x >= g.visible_nc) return;
  const bool simd = x < g.simd_end;
  const size_t plane = (size_t)g.rows * PW;
  const size_t col = (size_t)blockIdx.z * plane + __ldg(colidx + x);
  const unsigned char *p0 = srgb + lead + (c + 1) * 3 + (4 * rg + 1) * FP_RB;
#pragma unroll
  for (int j = 0; j < 4; j++) {
    const int y = y0 + 4 * rg + j;
    if (y >= g.visible_nr) break;
    const unsigned char *p = p0 + j * FP_RB;
    int bx = 0, by = 0, bl = -1;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      const int dx = (int)p[3 + ch] - (int)p[-3 + ch];
      const int dy = (int)p[FP_RB + ch] - (int)p[-FP_RB + ch];
      const int l = dx * dx + dy * dy;
      const bool take = (ch == 0) || (simd ? !(bl > l) : (l > bl));
      if (take) { bx = dx; by = dy; bl = l; }
    }
    const int o = __ldg(lut + ((by + 255) << 9) + (bx + 255));
    const size_t idx = col + (size_t)y * PW;
    vmag[idx] = __fsqrt_rn((float)bl);
    obin[idx] = (unsigned char)o;
  }
}

// cell_size == 8 (the default): same arithmetic, thread mapping chosen for the stores.  A tile is 256 x 16
// pixels; warp w owns the columns of one cell phase (x0 + w, x0 + w + 8, ...), lane l the l-th cell of the tile,
// so a warp's 32 outputs of a row are 32 CONSECUTIVE entries of the de-interleaved planes: one full 32-byte
// sector of orientation bytes and four of magnitudes per store instruction (the generic mapping scatters every
// store over 8 sectors).  A thread walks its column down the 16 rows.
constexpr int P8_TW = 256, P8_TH = 16;
constexpr int P8_RB = ((P8_TW + 2) * 3 + 15) & ~15;        // 784 staged bytes per row
__global__ void __launch_bounds__(256)
fhog_pixel8_kernel(const unsigned char *__restrict__ frames, float *__restrict__ vmag, unsigned char *__restrict__ obin,
                   FhogGeom g, const int *__restrict__ colidx, int PW, const unsigned char *__restrict__ lut) {
  __shared__ __align__(16) unsigned char srgb[(P8_TH + 2) * P8_RB];
  const int x0 = 1 + blockIdx.x * P8_TW, y0 = 1 + blockIdx.y * P8_TH;
  const unsigned char *src = frames + (size_t)blockIdx.z * g.rows * g.cols * 3;
  const int b0 = (x0 - 1) * 3, rowlimit = g.cols * 3;        // b0 = 768 * blockIdx.x: 16-byte aligned, like every row start
  for (int i = threadIdx.x; i < (P8_TH + 2) * (P8_RB / 16); i += 256) {
    const int r = i / (P8_RB / 16), q = i - r * (P8_RB / 16);
    const int gy = min(y0 - 1 + r, g.rows - 1), gb = b0 + 16 * q;
    const unsigned char *row = src + (size_t)gy * rowlimit;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (gb + 16 <= rowlimit) v = __ldg(reinterpret_cast<const uint4 *>(row + gb));
    else if (gb < rowlimit) {     // chunk crosses the end of the row: bytes past it are never read by a voter
      unsigned w[4];
#pragma unroll
      for (int k = 0; k < 4; k++) w[k] = gb + 4 * k + 4 <= rowlimit ? __ldg(reinterpret_cast<const unsigned *>(row + gb + 4 * k)) : 0u;
      v = make_uint4(w[0], w[1], w[2], w[3]);
    }
    reinterpret_cast<uint4 *>(srgb)[i] = v;
  }
  __syncthreads();
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  const int c = 8 * l + w, x = x0 + c;
  if (x >= g.visible_nc) return;
  const bool simd = x < g.simd_end;
  const size_t plane = (size_t)g.rows * PW;
  size_t idx = (size_t)blockIdx.z * plane + (size_t)y0 * PW + __ldg(colidx + x);
  const int nrow = min(P8_TH, g.visible_nr - y0);
  // The 9 bytes (left, centre, right pixel x RGB) of a row sit at byte 3c of the staged row: three aligned 4-byte words
  // and two funnel shifts deliver them (the shift 3c mod 4 = 3w mod 4 is warp uniform) instead of nine byte loads; the
  // centre bytes are reused as the "up" / "down" neighbours of the rows above and below.
  const unsigned *wrow = reinterpret_cast<const unsigned *>(srgb) + ((3 * c) >> 2);
  const int sh = ((3 * c) & 3) * 8;
  auto triple = [&](int r, unsigned &lo, unsigned &hi, unsigned &last) {   // bytes 0-3, 4-7, 8 of the 9
    const unsigned *q = wrow + r * (P8_RB / 4);
    const unsigned w0 = q[0], w1 = q[1], w2 = q[2];
    lo = __funnelshift_r(w0, w1, sh);
    hi = __funnelshift_r(w1, w2, sh);
    last = (w2 >> sh) & 0xffu;
  };
  auto byte_of = [](unsigned x, int k) -> int { return (int)__byte_perm(x, 0u, 0x4440 + k); };
  unsigned lo, hi, last;
  triple(0, lo, hi, last);
  int upc[3] = {byte_of(lo, 3), byte_of(hi, 0), byte_of(hi, 1)};          // centre pixel of the row above
  triple(1, lo, hi, last);
  for (int j = 0; j < nrow; j++, idx += PW) {
    const int lf[3] = {byte_of(lo, 0), byte_of(lo, 1), byte_of(lo, 2)};
    const int ce[3] = {byte_of(lo, 3), byte_of(hi, 0), byte_of(hi, 1)};
    const int rt[3] = {byte_of(hi, 2), byte_of(hi, 3), (int)last};
    triple(j + 2, lo, hi, last);                                         // the row below becomes the next current row
    const int dn[3] = {byte_of(lo, 3), byte_of(hi, 0), byte_of(hi, 1)};
    int bx = 0, by = 0, bl = -1;
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
      const int dx = rt[ch] - lf[ch];
      const int dy = dn[ch] - upc[ch];
      const int len = dx * dx + dy * dy;
      const bool take = (ch == 0) || (simd ? !(bl > len) : (len > bl));
      if (take) { bx = dx; by = dy; bl = len; }
    }
    vmag[idx] = __fsqrt_rn((float)bl);
    obin[idx] = __ldg(lut + ((by + 255) << 9) + (bx + 255));      // (a shared-memory copy of the table's centre measured slower: 1.39 vs 1.23 ms per 16 frames)
    upc[0] = ce[0]; upc[1] = ce[1]; upc[2] = ce[2];
  }
}

// ---- pass 2: one thread per histogram cell replays that cell's votes in raster order into a
// private shared-memory histogram (bank = thread, conflict-free); bit-identical to the reference.
__global__ void __launch_bounds__(FC_NT)
fhog_cell_kernel(const float *__restrict__ vmag, const unsigned char *__restrict__ obin, float *__restrict__ hist,
                 FhogGeom g, FhogTables tb, const int *__restrict__ colidx, int PW, int KW /* cached x weights per thread */) {
  extern __shared__ float sh[];          // [18][FC_NT] histogram, then [KW][FC_NT] x weights
  float *swx = sh + 18 * FC_NT;
  const int HR = g.cells_nr + 2, HC = g.cells_nc + 2;
  const int R = blockIdx.y, C = blockIdx.x * FC_NT + threadIdx.x;
#pragma unroll
  for (int o = 0; o < 18; o++) sh[o * FC_NT + threadIdx.x] = 0.f;
  if (C < HC) {
    const size_t plane = (size_t)g.rows * PW;
    const float *vin = vmag + (size_t)blockIdx.z * plane;
    const unsigned char *oin = obin + (size_t)blockIdx.z * plane;
    const int ya = tb.ylo[R], yb = tb.yhi[R], xa = tb.xlo[C], xb = tb.xhi[C];
    float *h = sh + threadIdx.x;
    float *wxs = swx + threadIdx.x;
    int *sidx = reinterpret_cast<int *>(swx + (size_t)KW * FC_NT) + threadIdx.x;
    const int nxw = min(xb - xa, KW);
    // per-thread tables over the cell's columns: x weight (sign bit = scalar-tail product order) and the
    // offset of column xa+k inside a de-interleaved plane row
    {
      const int NCB = PW / g.cell;
      int ph = xa % g.cell, q = xa / g.cell;
      for (int k = 0; k < nxw; k++) {
        const int x = xa + k;
        const float wx = (__ldg(tb.c0 + x) == C) ? __ldg(tb.vx1 + x) : __ldg(tb.vx0 + x);
        wxs[k * FC_NT] = (x < g.simd_end) ? wx : -wx;
        sidx[k * FC_NT] = ph * NCB + q;
        if (++ph == g.cell) { ph = 0; q++; }
      }
    }
    const int nfull = (xb - xa <= KW) ? nxw : 0;               // table-driven fast loop when the range is cached
    for (int y = ya; y < yb; y++) {
      const float wy = (__ldg(tb.r0 + y) == R) ? __ldg(tb.vy1 + y) : __ldg(tb.vy0 + y);
      const float *vrow = vin + (size_t)y * PW;
      const unsigned char *orow = oin + (size_t)y * PW;
      int k = 0;
      for (; k + 8 <= nfull; k += 8) {                          // 8 independent loads in flight, then 8 sequential adds
        float v[8]; int o[8];
#pragma unroll
        for (int j = 0; j < 8; j++) { const int idx = sidx[(k + j) * FC_NT]; v[j] = __ldg(vrow + idx); o[j] = (int)__ldg(orow + idx); }
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float wq = wxs[(k + j) * FC_NT];
          const float wx = fabsf(wq);
          // simd body: vy*(vx*v) (fhog.h:867-874) ; scalar tail: (vy*vx)*v (fhog.h:951-954)
          const float val = (__float_as_int(wq) < 0) ? __fmul_rn(__fmul_rn(wy, wx), v[j]) : __fmul_rn(wy, __fmul_rn(wx, v[j]));
          h[o[j] * FC_NT] = __fadd_rn(h[o[j] * FC_NT], val);
        }
      }
      for (; k < nfull; k++) {
        const int idx = sidx[k * FC_NT];
        const float v = __ldg(vrow + idx); const int o = (int)__ldg(orow + idx);
        const float wq = wxs[k * FC_NT], wx = fabsf(wq);
        const float val = (__float_as_int(wq) < 0) ? __fmul_rn(__fmul_rn(wy, wx), v) : __fmul_rn(wy, __fmul_rn(wx, v));
        h[o * FC_NT] = __fadd_rn(h[o * FC_NT], val);
      }
      if (!nfull) {                                             // very large cells: no tables, direct evaluation
        const int NCB = PW / g.cell;
        int ph = xa % g.cell, q = xa / g.cell;
        for (int x = xa; x < xb; x++) {
          const float wx = (__ldg(tb.c0 + x) == C) ? __ldg(tb.vx1 + x) : __ldg(tb.vx0 + x);
          const int idx = ph * NCB + q;
          const float v = __ldg(vrow + idx); const int o = (int)__ldg(orow + idx);
          const float val = (x < g.simd_end) ? __fmul_rn(wy, __fmul_rn(wx, v)) : __fmul_rn(__fmul_rn(wy, wx), v);
          h[o * FC_NT] = __fadd_rn(h[o * FC_NT], val);
          if (++ph == g.cell) { ph = 0; q++; }
        }
      }
    }
    float *dst = hist + ((size_t)blockIdx.z * HR * HC + (size_t)R * HC + C) * 18;
#pragma unroll
    for (int o = 0; o < 18; o++) dst[o] = h[o * FC_NT];
  }
}

__global__ void fhog_norm_kernel(const float *__restrict__ hist, float *__restrict__ norm, FhogGeom g) {
  int c = blockIdx.x * blockDim.x + threadIdx.x, r = blockIdx.y;
  if (c >= g.cells_nc) return;
  const int HC = g.cells_nc + 2;
  const float *h = hist + ((size_t)blockIdx.z * (g.cells_nr + 2) * HC + (size_t)(r + 1) * HC + (c + 1)) * 18;
  float n = 0.f;
#pragma unroll
  for (int o = 0; o < 9; o++) {
    float s = __fadd_rn(h[o], h[o + 9]);
    n = __fadd_rn(n, __fmul_rn(s, s));
  }
  norm[((size_t)blockIdx.z * g.cells_nr + r) * g.cells_nc + c] = n;
}

constexpr int FF_NT = 64;   // hog cells (consecutive columns of one row) per CTA
__global__ void __launch_bounds__(FF_NT)
fhog_feature_kernel(const float *__restrict__ hist, const float *__restrict__ norm, float *__restrict__ out, FhogGeom g) {
  // histograms in and features out are staged through shared memory so that both global streams are
  // contiguous (a row segment of 64 cells = 1152 floats in, 1984 floats out)
  __shared__ float sh[FF_NT * 18];
  __shared__ float so[FF_NT * 31];
  const int xb = blockIdx.x * FF_NT, y = blockIdx.y;
  const int ncell = min(FF_NT, g.hog_nc - xb);
  const int HC = g.cells_nc + 2;
  const float *hsrc = hist + ((size_t)blockIdx.z * (g.cells_nr + 2) * HC + (size_t)(y + 2) * HC + (xb + 2)) * 18;
  for (int i = threadIdx.x; i < ncell * 18; i += FF_NT) sh[i] = __ldg(hsrc + i);
  __syncthreads();
  const int t = threadIdx.x, x = xb + t;
  if (t < ncell) {
    const float *N = norm + (size_t)blockIdx.z * g.cells_nr * g.cells_nc;
#define NN(r, c) __ldg(N + (size_t)(r) * g.cells_nc + (c))
    const float n00 = NN(y, x), n01 = NN(y, x + 1), n02 = NN(y, x + 2), n10 = NN(y + 1, x), n11 = NN(y + 1, x + 1), n12 = NN(y + 1, x + 2),
                n20 = NN(y + 2, x), n21 = NN(y + 2, x + 1), n22 = NN(y + 2, x + 2);
#undef NN
    const float z1[4] = {n11, n01, n10, n00}, z2[4] = {n12, n02, n11, n01}, z3[4] = {n21, n11, n20, n10}, z4[4] = {n22, n12, n21, n11};
    float nn[4], n[4], tt[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      float s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(z1[k], z2[k]), z3[k]), z4[k]), 0.0001f);
      nn[k] = __fmul_rn(0.2f, __fsqrt_rn(s));
      n[k] = __fdiv_rn(0.1f, nn[k]);
    }
    float hv[18];
#pragma unroll
    for (int o = 0; o < 18; o++) hv[o] = sh[t * 18 + o];
    float *o31 = so + t * 31;
#pragma unroll
    for (int o = 0; o < 18; o += 3) {
      float hh[3][4];
#pragma unroll
      for (int j = 0; j < 3; j++) {
#pragma unroll
        for (int k = 0; k < 4; k++) hh[j][k] = __fmul_rn(hv[o + j] < nn[k] ? hv[o + j] : nn[k], n[k]);
        o31[o + j] = __fadd_rn(__fadd_rn(hh[j][0], hh[j][2]), __fadd_rn(hh[j][1], hh[j][3]));
      }
#pragma unroll
      for (int k = 0; k < 4; k++) tt[k] = __fadd_rn(tt[k], __fadd_rn(__fadd_rn(hh[0][k], hh[1][k]), hh[2][k]));
    }
    const float tscale = (float)(2 * 0.2357);
#pragma unroll
    for (int k = 0; k < 4; k++) tt[k] = __fmul_rn(tt[k], tscale);
#pragma unroll
    for (int o = 0; o < 9; o++) {
      float tmp = __fadd_rn(hv[o], hv[o + 9]), hk[4];
#pragma unroll
      for (int k = 0; k < 4; k++) hk[k] = __fmul_rn(tmp < nn[k] ? tmp : nn[k], n[k]);
      o31[18 + o] = __fadd_rn(__fadd_rn(hk[0], hk[2]), __fadd_rn(hk[1], hk[3]));
    }
#pragma unroll
    for (int k = 0; k < 4; k++) o31[27 + k] = tt[k];
  }
  __syncthreads();
  float *dst = out + (((size_t)blockIdx.z * g.out_nr + (y + g.pad_r)) * g.out_nc + (xb + g.pad_c)) * 31;
  for (int i = threadIdx.x; i < ncell * 31; i += FF_NT) dst[i] = so[i];
}

// ------------------------------------------------------------------------------------------ cell_size == 1
// dlib's separate routine (impl_extract_fhog_features_cell_size_1, fhog.h:495-694): every interior pixel is
// its own cell.  Pass 1 stores the SQUARED gradient length of the strongest channel (float) and the 18-way
// orientation of every interior pixel (border: 0, zero_border_pixels fhog.h:545); pass 2 turns the 3x3 block of
// norms around a pixel into the six non-zero features of its 31-vector (the others stay 0:
// init_hog_zero_everything, fhog.h:473-491).
__global__ void __launch_bounds__(256)
fhog1_pixel_kernel(const unsigned char *__restrict__ frames, float *__restrict__ norm, unsigned char *__restrict__ angle,
                   FhogGeom g, const unsigned char *__restrict__ lut) {
  const int x = blockIdx.x * 64 + (threadIdx.x & 63), y = blockIdx.y * 4 + (threadIdx.x >> 6);
  if (x >= g.cols || y >= g.rows) return;
  const size_t px = (size_t)blockIdx.z * g.rows * g.cols + (size_t)y * g.cols + x;
  if (x < 1 || y < 1 || x >= g.visible_nc || y >= g.visible_nr) { norm[px] = 0.f; angle[px] = 0; return; }
  const unsigned char *p = frames + px * 3;
  const int rs = g.cols * 3;
  const bool simd = x < g.simd_end;
  int bx = 0, by = 0, bl = -1;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    const int dx = (int)__ldg(p + 3 + ch) - (int)__ldg(p - 3 + ch);
    const int dy = (int)__ldg(p + rs + ch) - (int)__ldg(p - rs + ch);
    const int l = dx * dx + dy * dy;
    const bool take = (ch == 0) || (simd ? !(bl > l) : (l > bl));     // SIMD body keeps the later channel on ties, the scalar tail the earlier
    if (take) { bx = dx; by = dy; bl = l; }
  }
  norm[px] = (float)bl;
  angle[px] = __ldg(lut + ((by + 255) << 9) + (bx + 255));
}

constexpr int F1_NT = 64;
__global__ void __launch_bounds__(F1_NT)
fhog1_feature_kernel(const float *__restrict__ norm, const unsigned char *__restrict__ angle, float *__restrict__ out, FhogGeom g) {
  __shared__ float sn[3][F1_NT + 2];
  __shared__ float so[F1_NT * 31];
  const int xb = blockIdx.x * F1_NT, y = blockIdx.y;
  const int ncell = min(F1_NT, g.hog_nc - xb);
  const float *N = norm + (size_t)blockIdx.z * g.rows * g.cols;
  for (int i = threadIdx.x; i < 3 * (ncell + 2); i += F1_NT) {
    const int r = i / (ncell + 2), c = i - r * (ncell + 2);
    sn[r][c] = __ldg(N + (size_t)(y + r) * g.cols + xb + c);
  }
  for (int i = threadIdx.x; i < ncell * 31; i += F1_NT) so[i] = 0.f;
  __syncthreads();
  const int t = threadIdx.x;
  if (t < ncell) {
    const float n00 = sn[0][t], n01 = sn[0][t + 1], n02 = sn[0][t + 2], n10 = sn[1][t], n11 = sn[1][t + 1], n12 = sn[1][t + 2],
                n20 = sn[2][t], n21 = sn[2][t + 1], n22 = sn[2][t + 2];
    const float z1[4] = {n11, n01, n10, n00}, z2[4] = {n12, n02, n11, n01}, z3[4] = {n21, n11, n20, n10}, z4[4] = {n22, n12, n21, n11};
    const float temp0 = __fsqrt_rn(n11);
    float h0[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(z1[k], z2[k]), z3[k]), z4[k]), 0.0001f);
      const float nn = __fmul_rn(0.2f, __fsqrt_rn(s));
      const float n = __fdiv_rn(0.1f, nn);
      h0[k] = __fmul_rn(temp0 < nn ? temp0 : nn, n);                    // min(temp0, nn) * n
    }
    const float vv = __fadd_rn(__fadd_rn(h0[0], h0[2]), __fadd_rn(h0[1], h0[3]));   // sum(simd4f), SSE2 order
    const float tscale = (float)(2 * 0.2357);
    const int a = __ldg(angle + (size_t)blockIdx.z * g.rows * g.cols + (size_t)(y + 1) * g.cols + xb + t + 1);
    float *o31 = so + t * 31;
    o31[a] = vv;
    o31[a % 9 + 18] = vv;
#pragma unroll
    for (int k = 0; k < 4; k++) o31[27 + k] = __fmul_rn(__fadd_rn(0.f, h0[k]), tscale);
  }
  __syncthreads();
  float *dst = out + (((size_t)blockIdx.z * g.out_nr + (y + g.pad_r)) * g.out_nc + (xb + g.pad_c)) * 31;
  for (int i = threadIdx.x; i < ncell * 31; i += F1_NT) dst[i] = so[i];
}

// ------------------------------------------------------------------------------------------ host
size_t fhog_scratch_bytes(int n_frames, const FhogGeom &g) {
  if (g.cell == 1) return align256((size_t)n_frames * g.rows * g.cols * 4) + align256((size_t)n_frames * g.rows * g.cols) + (1 << 16);
  size_t hist = (size_t)n_frames * (g.cells_nr + 2) * (g.cells_nc + 2) * 18 * 4;
  size_t norm = (size_t)n_frames * g.cells_nr * g.cells_nc * 4;
  size_t tabs = (size_t)(g.rows + g.cols) * (2 + 4 + 4) + (size_t)(g.cells_nr + g.cells_nc + 4) * 8 + 4096;
  size_t vplane = (size_t)g.rows * (size_t)(g.cell * (g.cols / g.cell + 2)) * n_frames;
  return align256(hist) + align256(norm) + align256(vplane * 4) + align256(vplane) + 12 * align256(tabs) + (1 << 16);
}

// Vote tables for one geometry, built with the reference's float expressions and cached in the context
// (one device block; rebuilt only when rows / cols / cell change, so steady-state calls upload nothing
// and never synchronise).
struct FhogTabDev { FhogTables tb; const int *colidx; int KW; };

static int fhog_tables(b2f_ctx *ctx, const FhogGeom &g, cudaStream_t st, FhogTabDev &out) {
  const int cell = g.cell, HR = g.cells_nr + 2, HC = g.cells_nc + 2;
  const size_t o_r0 = 0, o_c0 = align256(o_r0 + 2 * (size_t)g.rows), o_vy0 = align256(o_c0 + 2 * (size_t)g.cols),
               o_vy1 = align256(o_vy0 + 4 * (size_t)g.rows), o_vx0 = align256(o_vy1 + 4 * (size_t)g.rows),
               o_vx1 = align256(o_vx0 + 4 * (size_t)g.cols), o_ylo = align256(o_vx1 + 4 * (size_t)g.cols),
               o_yhi = align256(o_ylo + 4 * (size_t)HR), o_xlo = align256(o_yhi + 4 * (size_t)HR), o_xhi = align256(o_xlo + 4 * (size_t)HC),
               o_col = align256(o_xhi + 4 * (size_t)HC), total = align256(o_col + 4 * (size_t)g.cols);
  auto bind = [&](char *base) {
    out.tb = FhogTables{(const short *)(base + o_r0), (const short *)(base + o_c0), (const float *)(base + o_vy0), (const float *)(base + o_vy1),
                        (const float *)(base + o_vx0), (const float *)(base + o_vx1), (const int *)(base + o_ylo), (const int *)(base + o_yhi),
                        (const int *)(base + o_xlo), (const int *)(base + o_xhi)};
    out.colidx = (const int *)(base + o_col);
  };
  if (ctx->fhog_tab && ctx->fhog_tab_key[0] == g.rows && ctx->fhog_tab_key[1] == g.cols && ctx->fhog_tab_key[2] == cell) {
    bind((char *)ctx->fhog_tab);
    out.KW = ctx->fhog_tab_kw;
    return B2F_OK;
  }
  std::vector<short> r0(g.rows, 0), c0(g.cols, 0);
  std::vector<float> vy0(g.rows, 0), vy1(g.rows, 0), vx0(g.cols, 0), vx1(g.cols, 0);
  for (int y = 1; y < g.visible_nr; y++) {                                   // fhog.h:823-826
    const float yp = ((float)y + 0.5) / (float)cell - 0.5;
    const int iyp = (int)std::floor(yp);
    const float a = yp - iyp;
    const float b = 1.0 - a;
    r0[y] = (short)(iyp + 1); vy0[y] = a; vy1[y] = b;
  }
  for (int x = 1; x < g.visible_nc; x++) {
    if (x < g.simd_end) {                                                    // fhog.h:838-841
      float xx = (float)x;
      float xp = (xx + 0.5f) / (float)cell + 0.5f;
      int ixp = (int)xp;
      float a = xp - (float)ixp;
      float b = 1.0f - a;
      c0[x] = (short)ixp; vx0[x] = a; vx1[x] = b;
    } else {                                                                 // fhog.h:946-949
      const float xp = ((double)x + 0.5) / (double)cell - 0.5;
      const int ixp = (int)std::floor(xp);
      const float a = xp - ixp;
      const float b = 1.0 - a;
      c0[x] = (short)(ixp + 1); vx0[x] = a; vx1[x] = b;
    }
  }
  std::vector<int> ylo(HR, 0), yhi(HR, 0), xlo(HC, 0), xhi(HC, 0);
  // [a[k], b[k]) = contiguous pixel range voting into histogram index k (pixel p votes into first[p]
  // and first[p]+1; first[] is non-decreasing).  Indices nobody votes into get an empty range placed
  // so that the span of any run of consecutive indices stays [a[first], b[last]).
  auto ranges = [](const std::vector<short> &first, int lo, int hi, std::vector<int> &a, std::vector<int> &b) {
    const int n = (int)a.size();
    for (int k = 0; k < n; k++) { a[k] = 1 << 30; b[k] = -1; }
    for (int p = lo; p < hi; p++)
      for (int k = first[p]; k <= first[p] + 1; k++)
        if (k >= 0 && k < n) { a[k] = std::min(a[k], p); b[k] = std::max(b[k], p + 1); }
    int kmin = -1, kmax = -1;
    for (int k = 0; k < n; k++) if (b[k] > a[k]) { if (kmin < 0) kmin = k; kmax = k; }
    if (kmin < 0) { for (int k = 0; k < n; k++) a[k] = b[k] = lo; return; }
    for (int k = 0; k < kmin; k++) a[k] = b[k] = a[kmin];
    for (int k = kmax + 1; k < n; k++) a[k] = b[k] = b[kmax];
  };
  ranges(r0, 1, std::max(g.visible_nr, 1), ylo, yhi);
  ranges(c0, 1, std::max(g.visible_nc, 1), xlo, xhi);
  const int NCB0 = g.cols / cell + 2;
  std::vector<int> colidx(g.cols);
  for (int x = 0; x < g.cols; x++) colidx[x] = (x % cell) * NCB0 + x / cell;      // cell-phase de-interleaved column
  int maxw = 1;
  for (int C = 0; C < HC; C++) maxw = std::max(maxw, xhi[C] - xlo[C]);

  // the previous block may still be read by kernels in flight: wait before replacing it
  B2F_CUDA(cudaStreamSynchronize(st));
  if (ctx->stream != st) B2F_CUDA(cudaStreamSynchronize(ctx->stream));
  ctx->fhog_tab_key[0] = ctx->fhog_tab_key[1] = ctx->fhog_tab_key[2] = 0;
  if (total > ctx->fhog_tab_cap) {
    if (ctx->fhog_tab) B2F_CUDA(cudaFree(ctx->fhog_tab));
    ctx->fhog_tab = nullptr; ctx->fhog_tab_cap = 0;
    void *pnew = nullptr;
    cudaError_t e = cudaMalloc(&pnew, total);
    if (e != cudaSuccess) { cudaGetLastError(); set_error("cudaMalloc(%zu bytes of FHOG tables) failed: %s", total, cudaGetErrorString(e)); return B2F_ENOMEM; }
    ctx->fhog_tab = pnew; ctx->fhog_tab_cap = total;
  }
  char *base = (char *)ctx->fhog_tab;
#define UP(off, v) B2F_CUDA(cudaMemcpyAsync(base + off, v.data(), v.size() * sizeof(v[0]), cudaMemcpyHostToDevice, st))
  UP(o_r0, r0); UP(o_c0, c0); UP(o_vy0, vy0); UP(o_vy1, vy1); UP(o_vx0, vx0); UP(o_vx1, vx1);
  UP(o_ylo, ylo); UP(o_yhi, yhi); UP(o_xlo, xlo); UP(o_xhi, xhi); UP(o_col, colidx);
#undef UP
  B2F_CUDA(cudaStreamSynchronize(st));   // host tables go out of scope at return
  ctx->fhog_tab_key[0] = g.rows; ctx->fhog_tab_key[1] = g.cols; ctx->fhog_tab_key[2] = cell;
  ctx->fhog_tab_kw = std::min(maxw, 96);
  bind(base);
  out.KW = ctx->fhog_tab_kw;
  return B2F_OK;
}

static int fhog_ensure_lut(b2f_ctx *ctx, cudaStream_t st) {
  if (ctx->fhog_lut) return B2F_OK;       // one-time 256 KB orientation table
  void *lut = nullptr;
  B2F_CUDA(cudaMalloc(&lut, 512 * 512));
  fhog_lut_kernel<<<dim3(2, 511), 256, 0, st>>>((unsigned char *)lut);
  B2F_LAUNCH_CHECK(ctx);
  ctx->fhog_lut = lut;
  return B2F_OK;
}

static int fhog1_device(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, const FhogGeom &g, float *d_out, cudaStream_t st) {
  const size_t px = (size_t)n_frames * g.rows * g.cols;
  float *norm = ctx->arena.get<float>(px);
  unsigned char *angle = ctx->arena.get<unsigned char>(px);
  B2F_ARENA_CHECK(ctx);
  int rc = fhog_ensure_lut(ctx, st);
  if (rc != B2F_OK) return rc;
  fhog1_pixel_kernel<<<dim3(ceil_div(g.cols, 64), ceil_div(g.rows, 4), n_frames), 256, 0, st>>>(d_frames, norm, angle, g, (const unsigned char *)ctx->fhog_lut);
  B2F_LAUNCH_CHECK(ctx);
  if (g.out_nr != g.hog_nr || g.out_nc != g.hog_nc)   // zero border of init_hog_zero_everything
    B2F_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * (size_t)n_frames * g.out_nr * g.out_nc * 31, st));
  fhog1_feature_kernel<<<dim3(ceil_div(g.hog_nc, F1_NT), g.hog_nr, n_frames), F1_NT, 0, st>>>(norm, angle, d_out, g);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

int fhog_device(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, const FhogGeom &g, float *d_out, cudaStream_t st) {
  if (g.cell == 1) return fhog1_device(ctx, d_frames, n_frames, g, d_out, st);
  const int cell = g.cell, HR = g.cells_nr + 2, HC = g.cells_nc + 2;
  FhogTabDev td;
  int trc = fhog_tables(ctx, g, st, td);
  if (trc != B2F_OK) return trc;
  const FhogTables tb = td.tb;
  const int *d_colidx = td.colidx;

  // ---- device buffers
  float *hist = ctx->arena.get<float>((size_t)n_frames * HR * HC * 18);
  float *norm = ctx->arena.get<float>((size_t)n_frames * g.cells_nr * g.cells_nc);
  const size_t vplane = (size_t)g.rows * (size_t)(cell * (g.cols / cell + 2));
  float *vmag = ctx->arena.get<float>((size_t)n_frames * vplane);
  unsigned char *obin = ctx->arena.get<unsigned char>((size_t)n_frames * vplane);
  B2F_ARENA_CHECK(ctx);

  const int NCB = g.cols / cell + 2, PW = cell * NCB;
  {
    int lrc = fhog_ensure_lut(ctx, st);
    if (lrc != B2F_OK) return lrc;
  }
  if (cell == 8 && g.cols % 16 == 0 && (reinterpret_cast<uintptr_t>(d_frames) & 15) == 0)
    fhog_pixel8_kernel<<<dim3(ceil_div(std::max(g.visible_nc - 1, 1), P8_TW), ceil_div(std::max(g.visible_nr - 1, 1), P8_TH), n_frames), 256, 0, st>>>(
        d_frames, vmag, obin, g, d_colidx, PW, (const unsigned char *)ctx->fhog_lut);
  else
  fhog_pixel_kernel<<<dim3(ceil_div(std::max(g.visible_nc - 1, 1), FP_TW), ceil_div(std::max(g.visible_nr - 1, 1), FP_TH), n_frames), FH_NT, 0, st>>>(
      d_frames, vmag, obin, g, d_colidx, PW, (const unsigned char *)ctx->fhog_lut,
      (g.cols % 16 == 0 && (reinterpret_cast<uintptr_t>(d_frames) & 15) == 0) ? 2 :
      (g.cols % 4 == 0 && (reinterpret_cast<uintptr_t>(d_frames) & 3) == 0) ? 1 : 0);
  B2F_LAUNCH_CHECK(ctx);
  {
    const int KW = td.KW;
    size_t smem = sizeof(float) * (size_t)(18 + 2 * KW) * FC_NT;   // histogram + x weights + column offsets
    B2F_CUDA(cudaFuncSetAttribute(fhog_cell_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fhog_cell_kernel<<<dim3(ceil_div(HC, FC_NT), HR, n_frames), FC_NT, smem, st>>>(vmag, obin, hist, g, tb, d_colidx, PW, KW);
    B2F_LAUNCH_CHECK(ctx);
  }
  fhog_norm_kernel<<<dim3(ceil_div(g.cells_nc, 128), g.cells_nr, n_frames), 128, 0, st>>>(hist, norm, g);
  B2F_LAUNCH_CHECK(ctx);
  if (g.out_nr != g.hog_nr || g.out_nc != g.hog_nc)   // zero border of init_hog (fhog.h:459-470)
    B2F_CUDA(cudaMemsetAsync(d_out, 0, sizeof(float) * (size_t)n_frames * g.out_nr * g.out_nc * 31, st));
  fhog_feature_kernel<<<dim3(ceil_div(g.hog_nc, FF_NT), g.hog_nr, n_frames), FF_NT, 0, st>>>(hist, norm, d_out, g);
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

static int fhog_check(const char *who, int rows, int cols, int cell, int frp, int fcp) {
  if (rows <= 0 || cols <= 0) { set_error("%s: bad image size %dx%d", who, rows, cols); return B2F_EINVAL; }
  if (cell <= 0 || frp <= 0 || fcp <= 0) { set_error("%s: cell_size and the paddings must be > 0 (fhog.h:710-717)", who); return B2F_EINVAL; }
  return B2F_OK;
}

// geometry-free wrappers for features.cu (the combined Harris + Canny + FHOG batch)
size_t fhog_scratch_simple(int n_frames, int rows, int cols, int cell, int frp, int fcp, int *out_nr, int *out_nc) {
  FhogGeom g;
  if (!fhog_geometry(rows, cols, cell, frp, fcp, g)) { *out_nr = *out_nc = 0; return 0; }
  *out_nr = g.out_nr; *out_nc = g.out_nc;
  return fhog_scratch_bytes(n_frames, g);
}
int fhog_device_simple(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, int rows, int cols, int cell, int frp, int fcp,
                       float *d_out, cudaStream_t st) {
  FhogGeom g;
  if (!fhog_geometry(rows, cols, cell, frp, fcp, g)) return B2F_OK;
  return fhog_device(ctx, d_frames, n_frames, g, d_out, st);
}
int fhog_check_args(const char *who, int rows, int cols, int cell, int frp, int fcp) { return fhog_check(who, rows, cols, cell, frp, fcp); }

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_fhog_size(int rows, int cols, int cell_size, int frp, int fcp, int *hog_nr, int *hog_nc) {
  if (!hog_nr || !hog_nc) { set_error("b2f_fhog_size: NULL output"); return B2F_EINVAL; }
  int rc = fhog_check("b2f_fhog_size", rows, cols, cell_size, frp, fcp);
  if (rc != B2F_OK) return rc;
  FhogGeom g;
  fhog_geometry(rows, cols, cell_size, frp, fcp, g);
  *hog_nr = g.out_nr; *hog_nc = g.out_nc;
  return B2F_OK;
}

int b2f_fhog_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int rows, int cols, int cell_size, int frp, int fcp,
                 float *d_hog, void *stream) {
  if (!ctx || !d_frames || n_frames <= 0) { set_error("b2f_fhog_dev: bad argument"); return B2F_EINVAL; }
  int rc = fhog_check("b2f_fhog_dev", rows, cols, cell_size, frp, fcp);
  if (rc != B2F_OK) return rc;
  FhogGeom g;
  if (!fhog_geometry(rows, cols, cell_size, frp, fcp, g)) return B2F_OK;   // empty output
  if (!d_hog) { set_error("b2f_fhog_dev: NULL output"); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, fhog_scratch_bytes(n_frames, g))) != B2F_OK) return rc;
  return fhog_device(ctx, d_frames, n_frames, g, d_hog, st);
}

int b2f_fhog_batch(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int rows, int cols, int cell_size, int frp, int fcp,
                   float *hog) {
  if (!ctx || !frames || n_frames <= 0) { set_error("b2f_fhog_batch: bad argument"); return B2F_EINVAL; }
  int rc = fhog_check("b2f_fhog_batch", rows, cols, cell_size, frp, fcp);
  if (rc != B2F_OK) return rc;
  FhogGeom g;
  if (!fhog_geometry(rows, cols, cell_size, frp, fcp, g)) return B2F_OK;
  if (!hog) { set_error("b2f_fhog_batch: NULL output"); return B2F_EINVAL; }
  return features_batch("b2f_fhog_batch", ctx, frames, 3, n_frames, rows, cols, nullptr, 0, nullptr, nullptr, nullptr, nullptr,
                        nullptr, nullptr, nullptr, cell_size, frp, fcp, hog);
}

int b2f_fhog_host(b2f_ctx *ctx, const uint8_t *rgb, int rows, int cols, int cell_size, int frp, int fcp, float *hog) {
  return b2f_fhog_batch(ctx, rgb, 1, rows, cols, cell_size, frp, fcp, hog);
}

}  // extern "C"
