// darknet.cu — YOLO detection and ImageNet classification of image.darknet (darknet_test_detector and
// darknet_predict_classifier, src/__R_API_*.c), bit-identical to the reference built with gcc -O2 on x86-64.
// The reference convolves with im2col + gemm_nn (loop order i-k-j): every output is a strictly sequential fp32 sum over
// k = (channel, ky, kx) from +0, each product and add rounded on its own.  No other order gives its bits, so the
// convolutions run on the CUDA cores in exactly that order (no tensor cores, no split-K); DESIGN.md §4.13 and §5.
//   dn_ingest_kernel      u8 interleaved RGB -> the planar float network input: load_image_stb's u8/255. through a table,
//                         then resize_image's two bilinear passes (the row pass is recomputed for rows iy and iy+1).
//   dn_conv_kernel<..>    implicit GEMM, filters x (frame, pixel) tiles; weight and im2col slices of k staged in shared
//                         memory by cp.async, double-buffered; epilogue = batch norm in double, scale, bias, leaky.
//   dn_maxpool_kernel, dn_avgpool_kernel   forward_maxpool_layer / forward_avgpool_layer.
// softmax, region (flatten, logistic, softmax, get_region_boxes, do_nms_sort) and top_k run on the host, compiled with
// -ffp-contract=off against glibc's libm and qsort, on the few floats the last GPU layer leaves per frame.
#include "common.cuh"
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <string>
#include <vector>

namespace b2f {

constexpr size_t DN_CHUNK_SCRATCH = (size_t)2 << 30;      // scratch bytes one chunk of a host batch may use
constexpr int DN_THREADS = 256, DN_BK = 8, DN_MALIGN = 64;

struct DnLayer {
  int type = 0;
  int filters = 0, size = 0, stride = 1, pad = 0, bn = 0, act = 0;
  float temperature = 1.f;
  int classes = 0, coords = 0, num = 0, softmax = 0;
  std::vector<float> anchors;
  int K = 0, Kpad = 0, Mpad = 0;                       // conv: K = c size size; weights [Kpad][Mpad], zero padded
  size_t o_wt = 0, o_mean = 0, o_scale = 0, o_bias = 0, o_den = 0;   // offsets into the device block
  const float *wt = nullptr, *mean = nullptr, *scale = nullptr, *bias = nullptr;
  const double *den = nullptr;                         // sqrt((double)rolling_variance) + .000001f
};

}  // namespace b2f

struct b2f_darknet_model {
  int device = 0, net_w = 0, net_h = 0;
  std::vector<b2f::DnLayer> L;
  int n_gpu = 0;              // layers 0 .. n_gpu-1 run on the device (conv, maxpool, avgpool)
  int last = 0;               // the last layer that is not a cost layer: the network output
  int region = -1;            // index of the region layer, -1 without one
  int dims[3] = {0, 0, 0};
  void *mem = nullptr;
  const float *lut = nullptr;   // (float)(u8 / 255.) for u8 = 0..255
};

namespace b2f {

// ------------------------------------------------------------------------------------------------------ kernels --
// One thread per output value of [n][3][RH][RW]; the source frame is [ih][iw][3] u8.
__global__ void dn_ingest_kernel(const uint8_t *__restrict__ rgb, int iw, int ih, const float *__restrict__ lut,
                                 float *__restrict__ out, int RW, int RH, int n) {
  const long long total = (long long)n * 3 * RH * RW;
  const float w_scale = __fdiv_rn((float)(iw - 1), (float)(RW - 1));
  const float h_scale = __fdiv_rn((float)(ih - 1), (float)(RH - 1));
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(i % RW);
    long long t = i / RW;
    const int r = (int)(t % RH);
    t /= RH;
    const int k = (int)(t % 3);
    const int f = (int)(t / 3);
    const uint8_t *src = rgb + (size_t)f * iw * ih * 3 + k;
    // the row pass of resize_image at (c, y)
    auto part = [&](int y) -> float {
      const uint8_t *row = src + (size_t)y * iw * 3;
      if (c == RW - 1 || iw == 1) return lut[row[(size_t)(iw - 1) * 3]];
      const float sx = __fmul_rn((float)c, w_scale);
      const int ix = (int)sx;
      const float dx = __fsub_rn(sx, (float)ix);
      const int ix1 = min(ix + 1, iw - 1);          // sx < iw - 1 for c < RW - 1; the reference asserts it
      return __fadd_rn(__fmul_rn(__fsub_rn(1.f, dx), lut[row[(size_t)ix * 3]]), __fmul_rn(dx, lut[row[(size_t)ix1 * 3]]));
    };
    const float sy = __fmul_rn((float)r, h_scale);
    const int iy = (int)sy;
    const float dy = __fsub_rn(sy, (float)iy);
    float v = __fmul_rn(__fsub_rn(1.f, dy), part(iy));
    if (!(r == RH - 1 || ih == 1)) v = __fadd_rn(v, __fmul_rn(dy, part(min(iy + 1, ih - 1))));
    out[i] = v;
  }
}

struct DnConvArgs {
  const float *in;            // frame f at in + f * in_fstride, planar [C][H][W]
  long long in_fstride;
  const float *wt, *mean, *scale, *bias;
  const double *den;
  float *out;                 // [nf][M][OH][OW]
  int C, H, W, OH, OW, size, stride, pad, M, Mpad, K, Kpad, nf, bn, leaky;
};

__device__ __forceinline__ void dn_cp4(float *s, const float *g, bool pred) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(s);
  const int sz = pred ? 4 : 0;                     // src-size 0: the 4 bytes are zero-filled
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(sa), "l"(g), "r"(sz));
}
__device__ __forceinline__ void dn_cp16(float *s, const float *g) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(s);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(sa), "l"(g));
}

// A CTA computes BM filters x BN columns (column = frame * OH * OW + pixel) with 256 threads of TM x TN accumulators;
// a thread's filters are ty + i * BM / TM and its columns tx + j * BN / TN.  Each accumulator walks k = 0 .. Kpad-1 in
// order with acc = acc + w * x, both rounded.  Padded taps are gathered as +0 and multiplied like the reference's im2col
// zeros; the k >= K rows are 0 * +0 = +0, which leaves an accumulator that started at +0 unchanged (§5).
template <int BM, int BN, int TM, int TN>
__global__ void __launch_bounds__(DN_THREADS) dn_conv_kernel(const DnConvArgs a) {
  static_assert((BM / TM) * (BN / TN) == DN_THREADS, "256 threads");
  static_assert(DN_BK * BM / 4 <= DN_THREADS && BN <= DN_THREADS, "one weight vector and one column per thread");
  __shared__ __align__(16) float Ws[2][DN_BK][BM];
  __shared__ __align__(16) float Xs[2][DN_BK][BN];
  const int tid = threadIdx.x;
  const int tx = tid % (BN / TN), ty = tid / (BN / TN);
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int P = a.OH * a.OW, Ntot = a.nf * P, SS = a.size * a.size;
  // this thread's im2col column and its rows in each slice
  const int nl = tid % BN, r0 = tid / BN;
  constexpr int RSTEP = DN_THREADS / BN, XPER = DN_BK * BN / DN_THREADS;
  const int n = n0 + nl;
  const bool nvalid = n < Ntot;
  int iy0 = 0, ix0 = 0;
  const float *base = a.in;
  if (nvalid) {
    const int f = n / P, p = n - f * P, oy = p / a.OW, ox = p - oy * a.OW;
    iy0 = oy * a.stride - a.pad;
    ix0 = ox * a.stride - a.pad;
    base = a.in + f * a.in_fstride;
  }
  auto load = [&](int k0, int buf) {
    if (tid < DN_BK * BM / 4) {
      const int kk = tid / (BM / 4), mm = (tid % (BM / 4)) * 4;
      dn_cp16(&Ws[buf][kk][mm], a.wt + (size_t)(k0 + kk) * a.Mpad + m0 + mm);
    }
#pragma unroll
    for (int e = 0; e < XPER; e++) {
      const int kk = r0 + e * RSTEP, k = k0 + kk;
      bool ok = nvalid && k < a.K;
      const float *src = a.in;
      if (ok) {
        const int c = k / SS, r = k - c * SS, ky = r / a.size, kx = r - ky * a.size;
        const int iy = iy0 + ky, ix = ix0 + kx;
        ok = iy >= 0 && iy < a.H && ix >= 0 && ix < a.W;
        if (ok) src = base + ((size_t)c * a.H + iy) * a.W + ix;
      }
      dn_cp4(&Xs[buf][kk][nl], src, ok);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; i++)
#pragma unroll
    for (int j = 0; j < TN; j++) acc[i][j] = 0.f;
  const int nk = a.Kpad / DN_BK;
  load(0, 0);
  for (int t = 0; t < nk; t++) {
    const int buf = t & 1;
    if (t + 1 < nk) {
      load((t + 1) * DN_BK, buf ^ 1);
      asm volatile("cp.async.wait_group 1;\n" ::);
    } else {
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < DN_BK; kk++) {
      float wv[TM], xv[TN];
#pragma unroll
      for (int i = 0; i < TM; i++) wv[i] = Ws[buf][kk][ty + i * (BM / TM)];
#pragma unroll
      for (int j = 0; j < TN; j++) xv[j] = Xs[buf][kk][tx + j * (BN / TN)];
#pragma unroll
      for (int i = 0; i < TM; i++)
#pragma unroll
        for (int j = 0; j < TN; j++) acc[i][j] = __fadd_rn(acc[i][j], __fmul_rn(wv[i], xv[j]));
    }
    __syncthreads();
  }
  // forward_batchnorm_layer (normalize_cpu, scale_bias), add_bias, activate_array, in that order
#pragma unroll
  for (int i = 0; i < TM; i++) {
    const int m = m0 + ty + i * (BM / TM);
    if (m >= a.M) continue;
    const float mean = a.bn ? a.mean[m] : 0.f, scale = a.bn ? a.scale[m] : 0.f, bias = a.bias[m];
    const double den = a.bn ? a.den[m] : 1.0;
#pragma unroll
    for (int j = 0; j < TN; j++) {
      const int nn = n0 + tx + j * (BN / TN);
      if (nn >= Ntot) continue;
      float v = acc[i][j];
      if (a.bn) {
        v = __double2float_rn(__ddiv_rn((double)__fsub_rn(v, mean), den));
        v = __fmul_rn(v, scale);
      }
      v = __fadd_rn(v, bias);
      if (a.leaky && !(v > 0.f)) v = __double2float_rn(__dmul_rn(0.1, (double)v));
      const int f = nn / P, p = nn - f * P;
      a.out[((size_t)f * a.M + m) * P + p] = v;
    }
  }
}

__global__ void dn_maxpool_kernel(const float *__restrict__ in, float *__restrict__ out, int C, int H, int W, int OH, int OW,
                                  int size, int stride, int pad, long long total) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(i % OW);
    long long t = i / OW;
    const int y = (int)(t % OH);
    t /= OH;                                          // frame * C + channel
    const float *src = in + t * H * W;
    float mx = -FLT_MAX;
    for (int n = 0; n < size; n++)
      for (int m = 0; m < size; m++) {
        const int ch = y * stride + n - pad, cw = j * stride + m - pad;
        const float v = (ch >= 0 && ch < H && cw >= 0 && cw < W) ? src[(size_t)ch * W + cw] : -FLT_MAX;
        mx = (v > mx) ? v : mx;
      }
    out[i] = mx;
  }
}

__global__ void dn_avgpool_kernel(const float *__restrict__ in, float *__restrict__ out, int hw, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const float *src = in + (size_t)i * hw;
  float s = 0.f;
  for (int k = 0; k < hw; k++) s = __fadd_rn(s, src[k]);
  out[i] = __fdiv_rn(s, (float)hw);
}

// ------------------------------------------------------------------------------------------------- geometry ------
struct DnGeom {
  int RW = 0, RH = 0;             // the resized planes the ingest writes
  int nw = 0, nh = 0;             // the size layer 0 sees (a prefix of the planes when they are larger)
  std::vector<int> c, h, w, oc, oh, ow;
  size_t act = 0;                 // floats per frame of the largest GPU layer output
};

// mode 0 = detect, 1 = classify with resize, 2 = classify without (darknet_predict_classifier's resize_min)
static int dn_geom(const char *who, const b2f_darknet_model *m, int mode, int W, int H, DnGeom &g) {
  if (mode == 0) {
    g.RW = g.nw = m->net_w;
    g.RH = g.nh = m->net_h;
  } else {
    long long rw = W, rh = H;
    const int mn = m->net_w;
    if (rw < rh) { rh = rh * mn / rw; rw = mn; } else { rw = rw * mn / rh; rh = mn; }
    if (rw * rh * 3 > 2147483647LL) { set_error("%s: the %dx%d frame resizes to %lldx%lld, over the reference's int indexing", who, W, H, rw, rh); return B2F_EUNSUP; }
    g.RW = (int)rw; g.RH = (int)rh;
    if (mode == 1) { g.nw = g.RW; g.nh = g.RH; } else { g.nw = m->net_w; g.nh = m->net_h; }
    // resize = FALSE reads the first 3 net_w net_h floats of the resized planes; a cfg taller than wide can make them
    // shorter than that, and the reference then reads past its buffer: there is no answer to reproduce
    if ((long long)g.RW * g.RH < (long long)g.nw * g.nh) {
      set_error("%s: the %dx%d frame resizes to %dx%d, fewer floats than the %dx%d network reads without resize", who, W, H,
                g.RW, g.RH, g.nw, g.nh);
      return B2F_EUNSUP;
    }
  }
  int c = 3, h = g.nh, w = g.nw;
  const int nl = (int)m->L.size();
  g.c.resize(nl); g.h.resize(nl); g.w.resize(nl); g.oc.resize(nl); g.oh.resize(nl); g.ow.resize(nl);
  g.act = 0;
  for (int i = 0; i < nl; i++) {
    const DnLayer &L = m->L[i];
    g.c[i] = c; g.h[i] = h; g.w[i] = w;
    int oc = c, oh = h, ow = w;
    if (L.type == B2F_DN_CONV) {
      oc = L.filters;
      oh = (h + 2 * L.pad - L.size) / L.stride + 1;
      ow = (w + 2 * L.pad - L.size) / L.stride + 1;
    } else if (L.type == B2F_DN_MAXPOOL) {
      oh = (h + 2 * L.pad) / L.stride;
      ow = (w + 2 * L.pad) / L.stride;
    } else if (L.type == B2F_DN_AVGPOOL) {
      oh = ow = 1;
    }
    if (oh <= 0 || ow <= 0) { set_error("%s: layer %d has no output at a %dx%d network input", who, i, g.nw, g.nh); return B2F_EINVAL; }
    if (i < m->n_gpu) g.act = std::max(g.act, (size_t)oc * oh * ow);
    g.oc[i] = oc; g.oh[i] = oh; g.ow[i] = ow;
    c = oc; h = oh; w = ow;
  }
  return B2F_OK;
}

static size_t dn_scratch_bytes(const DnGeom &g, int n) {
  return align256((size_t)n * 3 * g.RW * g.RH * 4) + 2 * align256((size_t)n * std::max<size_t>(g.act, 1) * 4);
}

// ------------------------------------------------------------------------------------------------- forward ------
template <int BM, int BN, int TM, int TN>
static void dn_conv_launch(const DnConvArgs &a, cudaStream_t st) {
  const dim3 grid((unsigned)ceil_div(a.nf * a.OH * a.OW, BN), (unsigned)ceil_div(a.M, BM));
  dn_conv_kernel<BM, BN, TM, TN><<<grid, DN_THREADS, 0, st>>>(a);
}

// The tile is chosen from the layer shape: the largest whose grid still gives every SM two CTAs, since with no split-K
// the outputs are the only parallelism (the 13x13 layers of tiny-yolo-voc at batch 1 have 1024 x 169 of them).
static void dn_conv(const b2f_ctx *ctx, const DnConvArgs &a, cudaStream_t st) {
  const long long N = (long long)a.nf * a.OH * a.OW;
  auto ctas = [&](int bm, int bn) { return (long long)ceil_div(a.M, bm) * ((N + bn - 1) / bn); };
  const long long want = 2LL * ctx->sm_count;
  if (a.M <= 16) dn_conv_launch<16, 256, 2, 8>(a, st);
  else if (ctas(64, 128) >= want) dn_conv_launch<64, 128, 4, 8>(a, st);
  else if (ctas(32, 64) >= want) dn_conv_launch<32, 64, 2, 4>(a, st);
  else dn_conv_launch<32, 32, 2, 2>(a, st);
}

static unsigned dn_blocks(long long total) { return (unsigned)std::min<long long>((total + 255) / 256, 65536LL * 4); }

// n frames [n][H][W][3] u8 in HBM -> the device output of layer `upto` (-1: the network input), in *out.  The arena is
// reserved by the caller for dn_scratch_bytes(g, n).
static int dn_forward(b2f_ctx *ctx, const b2f_darknet_model *m, const DnGeom &g, const uint8_t *d_rgb, int n, int W, int H,
                      int upto, const float **out, cudaStream_t st) {
  float *input = ctx->arena.get<float>((size_t)n * 3 * g.RW * g.RH);
  float *act[2] = {ctx->arena.get<float>((size_t)n * std::max<size_t>(g.act, 1)), ctx->arena.get<float>((size_t)n * std::max<size_t>(g.act, 1))};
  B2F_ARENA_CHECK(ctx);
  const long long tot_in = (long long)n * 3 * g.RW * g.RH;
  dn_ingest_kernel<<<dn_blocks(tot_in), 256, 0, st>>>(d_rgb, W, H, m->lut, input, g.RW, g.RH, n);
  B2F_LAUNCH_CHECK(ctx);
  const float *cur = input;
  long long fstride = 3LL * g.RW * g.RH;
  for (int i = 0; i <= upto; i++) {
    const DnLayer &L = m->L[i];
    float *dst = act[i & 1];
    if (L.type == B2F_DN_CONV) {
      if ((long long)n * g.oh[i] * g.ow[i] > INT_MAX) {     // the kernel indexes the (frame, pixel) columns in int
        set_error("%d frames of %dx%d outputs at layer %d overflow the column index", n, g.ow[i], g.oh[i], i);
        return B2F_EUNSUP;
      }
      DnConvArgs a;
      a.in = cur; a.in_fstride = fstride;
      a.wt = L.wt; a.mean = L.mean; a.scale = L.scale; a.bias = L.bias; a.den = L.den;
      a.out = dst;
      a.C = g.c[i]; a.H = g.h[i]; a.W = g.w[i]; a.OH = g.oh[i]; a.OW = g.ow[i];
      a.size = L.size; a.stride = L.stride; a.pad = L.pad;
      a.M = L.filters; a.Mpad = L.Mpad; a.K = L.K; a.Kpad = L.Kpad; a.nf = n; a.bn = L.bn; a.leaky = L.act == B2F_DN_LEAKY;
      dn_conv(ctx, a, st);
    } else if (L.type == B2F_DN_MAXPOOL) {
      if (fstride != (long long)g.c[i] * g.h[i] * g.w[i]) { set_error("internal: maxpool over a strided input"); return B2F_EUNSUP; }
      const long long tot = (long long)n * g.oc[i] * g.oh[i] * g.ow[i];
      dn_maxpool_kernel<<<dn_blocks(tot), 256, 0, st>>>(cur, dst, g.c[i], g.h[i], g.w[i], g.oh[i], g.ow[i], L.size, L.stride, L.pad, tot);
    } else {                                          // avgpool
      if (fstride != (long long)g.c[i] * g.h[i] * g.w[i]) { set_error("internal: avgpool over a strided input"); return B2F_EUNSUP; }
      const int tot = n * g.c[i];
      dn_avgpool_kernel<<<ceil_div(tot, 256), 256, 0, st>>>(cur, dst, g.h[i] * g.w[i], tot);
    }
    B2F_LAUNCH_CHECK(ctx);
    cur = dst;
    fstride = (long long)g.oc[i] * g.oh[i] * g.ow[i];
  }
  *out = cur;
  return B2F_OK;
}

// ---------------------------------------------------------------------------------------------- host tails -----
// Written from the reference's operation order (blas.c softmax, activations.h logistic, region_layer.c, box.c); this
// file's host code is compiled with -ffp-contract=off, and exp is glibc's.
static float dn_logistic(float x) { return 1. / (1. + std::exp((double)-x)); }

static void dn_softmax(float *x, int n, float temp) {
  float sum = 0, largest = -FLT_MAX;
  for (int i = 0; i < n; ++i)
    if (x[i] > largest) largest = x[i];
  for (int i = 0; i < n; ++i) {
    const float e = std::exp((double)(x[i] / temp - largest / temp));
    sum += e;
    x[i] = e;
  }
  for (int i = 0; i < n; ++i) x[i] /= sum;
}

// forward_region_layer at inference: in = the previous layer's [n (classes + 5)][h][w] planes -> out (l.output)
static void dn_region_forward(const DnLayer &L, int lw, int lh, const float *in, float *out) {
  const int size = L.coords + L.classes + 1, sz = lw * lh, layers = size * L.num;
  for (int c = 0; c < layers; ++c)
    for (int i = 0; i < sz; ++i) out[i * layers + c] = in[c * sz + i];
  for (int i = 0; i < sz * L.num; ++i) out[size * i + 4] = dn_logistic(out[size * i + 4]);
  if (L.softmax)
    for (int i = 0; i < sz * L.num; ++i) dn_softmax(out + size * i + 5, L.classes, 1);
}

struct DnBox { float x, y, w, h; };
struct DnSortable { int index; int cls; float **probs; };     // box.c's sortable_bbox: the same size for qsort

static int dn_nms_comparator(const void *pa, const void *pb) {
  const DnSortable a = *(const DnSortable *)pa, b = *(const DnSortable *)pb;
  const float diff = a.probs[a.index][b.cls] - b.probs[b.index][b.cls];
  if (diff < 0) return 1;
  else if (diff > 0) return -1;
  return 0;
}
static float dn_overlap(float x1, float w1, float x2, float w2) {
  const float l1 = x1 - w1 / 2, l2 = x2 - w2 / 2, left = l1 > l2 ? l1 : l2;
  const float r1 = x1 + w1 / 2, r2 = x2 + w2 / 2, right = r1 < r2 ? r1 : r2;
  return right - left;
}
static float dn_iou(const DnBox &a, const DnBox &b) {
  const float w = dn_overlap(a.x, a.w, b.x, b.w), h = dn_overlap(a.y, a.h, b.y, b.h);
  const float i = (w < 0 || h < 0) ? 0 : w * h;
  const float u = a.w * a.h + b.w * b.h - i;
  return i / u;
}

// get_region_boxes(l, 1, 1, thresh, ..) + do_nms_sort(.., .4) + the count of darknet_test_detector, on l.output
static int dn_region_tail(const DnLayer &L, int lw, int lh, const float *pred, float thresh, float *probs, float *boxes_out) {
  const int total = lw * lh * L.num, np = L.classes + 1;
  std::vector<DnBox> boxes(total);
  std::vector<float *> rows(total);
  std::fill(probs, probs + (size_t)total * np, 0.f);
  for (int i = 0; i < lw * lh; ++i) {
    const int row = i / lw, col = i % lw;
    for (int n = 0; n < L.num; ++n) {
      const int index = i * L.num + n, bi = index * (L.classes + 5);
      const float scale = pred[bi + 4];
      DnBox &b = boxes[index];
      b.x = (col + dn_logistic(pred[bi + 0])) / lw;
      b.y = (row + dn_logistic(pred[bi + 1])) / lh;
      b.w = std::exp((double)pred[bi + 2]) * L.anchors[2 * n] / lw;
      b.h = std::exp((double)pred[bi + 3]) * L.anchors[2 * n + 1] / lh;
      float *p = probs + (size_t)index * np;
      rows[index] = p;
      for (int j = 0; j < L.classes; ++j) {
        const float prob = scale * pred[bi + 5 + j];
        p[j] = (prob > thresh) ? prob : 0;
      }
    }
  }
  const float nms = .4;
  std::vector<DnSortable> s(total);
  for (int i = 0; i < total; ++i) s[i] = DnSortable{i, 0, rows.data()};
  for (int k = 0; k < L.classes; ++k) {
    for (int i = 0; i < total; ++i) s[i].cls = k;
    qsort(s.data(), total, sizeof(DnSortable), dn_nms_comparator);
    for (int i = 0; i < total; ++i) {
      if (rows[s[i].index][k] == 0) continue;
      const DnBox a = boxes[s[i].index];
      for (int j = i + 1; j < total; ++j)
        if (dn_iou(a, boxes[s[j].index]) > nms) rows[s[j].index][k] = 0;
    }
  }
  int found = 0;
  for (int i = 0; i < total; ++i) {
    const float *p = rows[i];
    int mi = 0;
    float mx = p[0];
    for (int j = 1; j < L.classes; ++j)
      if (p[j] > mx) { mx = p[j]; mi = j; }
    if (p[mi] > thresh) found++;
    boxes_out[4 * i + 0] = boxes[i].x; boxes_out[4 * i + 1] = boxes[i].y;
    boxes_out[4 * i + 2] = boxes[i].w; boxes_out[4 * i + 3] = boxes[i].h;
  }
  return found;
}

static void dn_top_k(const float *a, int n, int k, int *index) {
  for (int j = 0; j < k; ++j) index[j] = -1;
  for (int i = 0; i < n; ++i) {
    int curr = i;
    for (int j = 0; j < k; ++j)
      if (index[j] < 0 || a[curr] > a[index[j]]) std::swap(curr, index[j]);
  }
}

// The host layers after the GPU prefix, on one frame: x = the last GPU layer's output -> the output of layer `upto`
// (softmax / region as the reference leaves l.output) in `out`.  Returns its length.
static size_t dn_host_layers(const b2f_darknet_model *m, const DnGeom &g, const float *x, int upto, std::vector<float> &out) {
  size_t len = (size_t)g.oc[m->n_gpu - 1] * g.oh[m->n_gpu - 1] * g.ow[m->n_gpu - 1];
  out.assign(x, x + len);
  std::vector<float> tmp;
  for (int i = m->n_gpu; i <= upto; i++) {
    const DnLayer &L = m->L[i];
    if (L.type == B2F_DN_SOFTMAX) {
      dn_softmax(out.data(), (int)len, L.temperature);
    } else if (L.type == B2F_DN_REGION) {
      tmp.resize(len);
      dn_region_forward(L, g.w[i], g.h[i], out.data(), tmp.data());
      out.swap(tmp);
    }
  }
  return len;
}

static int dn_check(const char *who, const b2f_darknet_model *m, int n, int W, int H) {
  if (!m) { set_error("%s: NULL model", who); return B2F_EINVAL; }
  if (n <= 0 || W <= 0 || H <= 0) { set_error("%s: bad size %d x %dx%d", who, n, W, H); return B2F_EINVAL; }
  if ((long long)W * H * 3 > 2147483647LL) { set_error("%s: %dx%d overflows the int indexing of the reference", who, W, H); return B2F_EUNSUP; }
  return B2F_OK;
}

// Forward pass of n device frames to the last GPU layer, and its output on the host: x [n][len].
static int dn_run_to_host(b2f_ctx *ctx, const b2f_darknet_model *m, const DnGeom &g, const uint8_t *d_rgb, int n, int W, int H,
                          std::vector<float> &x, size_t &len, cudaStream_t st) {
  const size_t mark = ctx->arena.off;
  const float *d_out = nullptr;
  int rc = dn_forward(ctx, m, g, d_rgb, n, W, H, m->n_gpu - 1, &d_out, st);
  ctx->arena.off = mark;
  if (rc != B2F_OK) return rc;
  const int l = m->n_gpu - 1;
  len = (size_t)g.oc[l] * g.oh[l] * g.ow[l];
  x.resize((size_t)n * len);
  B2F_CUDA(cudaMemcpyAsync(x.data(), d_out, x.size() * 4, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  return B2F_OK;
}

struct DnDetectOut { float thresh; float *probs, *boxes; int *count; };
struct DnClassifyOut { int resize, top; int *index; double *prob; };

static int dn_detect_frames(b2f_ctx *ctx, const b2f_darknet_model *m, const DnGeom &g, const uint8_t *d_rgb, int n, int W, int H,
                            const DnDetectOut &o, cudaStream_t st) {
  std::vector<float> x, y;
  size_t len;
  int rc = dn_run_to_host(ctx, m, g, d_rgb, n, W, H, x, len, st);
  if (rc != B2F_OK) return rc;
  const int r = m->region;
  const size_t total = (size_t)m->dims[0], np = (size_t)m->dims[1] + 1;
  for (int f = 0; f < n; f++) {
    dn_host_layers(m, g, x.data() + (size_t)f * len, r, y);
    o.count[f] = dn_region_tail(m->L[r], g.w[r], g.h[r], y.data(), o.thresh, o.probs + f * total * np, o.boxes + f * total * 4);
  }
  return B2F_OK;
}

static int dn_classify_frames(b2f_ctx *ctx, const b2f_darknet_model *m, const DnGeom &g, const uint8_t *d_rgb, int n, int W, int H,
                              const DnClassifyOut &o, cudaStream_t st) {
  std::vector<float> x, y;
  size_t len;
  int rc = dn_run_to_host(ctx, m, g, d_rgb, n, W, H, x, len, st);
  if (rc != B2F_OK) return rc;
  std::vector<int> idx(o.top);
  for (int f = 0; f < n; f++) {
    const size_t outn = dn_host_layers(m, g, x.data() + (size_t)f * len, m->last, y);
    if (outn != (size_t)m->dims[2]) {
      set_error("classify: the network output has %zu values at this frame size, net.outputs is %d", outn, m->dims[2]);
      return B2F_EUNSUP;
    }
    dn_top_k(y.data(), m->dims[2], o.top, idx.data());
    for (int i = 0; i < o.top; i++) {
      o.index[(size_t)f * o.top + i] = idx[i];
      o.prob[(size_t)f * o.top + i] = y[idx[i]];
    }
  }
  return B2F_OK;
}

// The chunked host batch shared by detect and classify: chunk c+1 uploads (copy-in stream) while chunk c runs.
template <typename Run>
static int dn_batch(const char *who, b2f_ctx *ctx, const DnGeom &g, const uint8_t *frames, int n_frames, int W, int H, Run run) {
  B2F_CUDA(cudaSetDevice(ctx->device));
  const size_t fb = (size_t)W * H * 3;
  const size_t per = dn_scratch_bytes(g, 1) + 2 * fb;
  const int C = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, DN_CHUNK_SCRATCH / per));
  int rc;
  if ((rc = arena_reserve(ctx, dn_scratch_bytes(g, C) + 2 * align256(fb * C))) != B2F_OK) return rc;
  uint8_t *d_in[2] = {ctx->arena.get<uint8_t>(fb * C), ctx->arena.get<uint8_t>(fb * C)};
  B2F_ARENA_CHECK(ctx);
  cudaStream_t st = ctx->stream;
  const int NCH = ceil_div(n_frames, C);
  if ((rc = pipe_prepare(ctx, NCH)) != B2F_OK) return rc;
  auto upload = [&](int c) -> int {
    const int f0 = c * C, nf = std::min(C, n_frames - f0);
    if (cudaMemcpyAsync(d_in[c & 1], frames + fb * f0, fb * nf, cudaMemcpyHostToDevice, ctx->s_in) != cudaSuccess ||
        cudaEventRecord(ctx->events[c], ctx->s_in) != cudaSuccess) return B2F_ECUDA;
    return B2F_OK;
  };
  rc = upload(0);
  for (int c = 0; c < NCH && rc == B2F_OK; c++) {
    const int f0 = c * C, nf = std::min(C, n_frames - f0);
    if (cudaStreamWaitEvent(st, ctx->events[c], 0) != cudaSuccess) { rc = B2F_ECUDA; break; }
    // chunk c+1 overwrites the buffer chunk c-1 read: that chunk's kernels finished before its tail ran
    if (c + 1 < NCH && (rc = upload(c + 1)) != B2F_OK) break;
    rc = run(d_in[c & 1], f0, nf, st);
  }
  if (rc == B2F_ECUDA && cudaPeekAtLastError() != cudaSuccess) set_error("%s: %s", who, cudaGetErrorString(cudaGetLastError()));
  const int rd = pipe_drain(ctx);
  return rc != B2F_OK ? rc : rd;
}

static int dn_check_detect(const char *who, const b2f_darknet_model *m) {
  if (m->region < 0) { set_error("%s: the network has no region layer", who); return B2F_EINVAL; }
  return B2F_OK;
}
static int dn_check_classify(const char *who, const b2f_darknet_model *m, int top) {
  if (m->region >= 0) { set_error("%s: the network ends in a region layer (use detect)", who); return B2F_EINVAL; }
  if (top < 1 || top > m->dims[2]) { set_error("%s: top %d is outside 1..%d", who, top, m->dims[2]); return B2F_EINVAL; }
  return B2F_OK;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_darknet_model_create(b2f_ctx *ctx, const b2f_darknet_layer *layers, int n_layers, int net_w, int net_h,
                             b2f_darknet_model **model) {
  const char *who = "b2f_darknet_model_create";
  if (!ctx || !layers || !model) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  *model = nullptr;
  if (n_layers <= 0) { set_error("%s: %d layers", who, n_layers); return B2F_EINVAL; }
  if (net_w < 2 || net_h < 2) { set_error("%s: network size %dx%d (at least 2x2)", who, net_w, net_h); return B2F_EINVAL; }
  b2f_darknet_model *m = new b2f_darknet_model();
  m->device = ctx->device;
  m->net_w = net_w;
  m->net_h = net_h;
  m->L.resize(n_layers);
  auto fail = [&](const char *fmt, int l, const char *what) {
    std::string f = std::string("%s: layer %d (%s): ") + fmt;
    set_error(f.c_str(), who, l, what ? what : "?");
    delete m;
    return B2F_EINVAL;
  };
  bool host_part = false;
  m->n_gpu = 0;
  int c = 3, h = net_h, w = net_w;
  for (int l = 0; l < n_layers; l++) {
    const b2f_darknet_layer &S = layers[l];
    DnLayer &L = m->L[l];
    const char *nm = S.name;
    L.type = S.type;
    switch (S.type) {
      case B2F_DN_CONV:
      case B2F_DN_MAXPOOL:
      case B2F_DN_AVGPOOL:
        if (host_part) return fail("a GPU layer after a softmax or region layer is not supported", l, nm);
        m->n_gpu = l + 1;
        break;
      case B2F_DN_SOFTMAX:
      case B2F_DN_REGION:
        if (l == 0) return fail("the first layer must be a convolutional or pooling layer", l, nm);
        if (host_part) return fail("only cost layers may follow a softmax, region or cost layer", l, nm);
        host_part = true;
        break;
      case B2F_DN_COST:
        if (l == 0) return fail("the first layer must be a convolutional or pooling layer", l, nm);
        host_part = true;
        break;
      default:
        return fail("this layer type is not supported", l, nm);
    }
    int oc = c, oh = h, ow = w;
    if (S.type == B2F_DN_CONV) {
      if (S.filters <= 0 || S.size <= 0 || S.stride <= 0 || S.pad < 0) return fail("bad filters, size, stride or pad", l, nm);
      if (S.activation != B2F_DN_LINEAR && S.activation != B2F_DN_LEAKY) return fail("only leaky and linear activations are supported", l, nm);
      if (!S.biases || !S.weights || (S.batch_normalize && (!S.scales || !S.rolling_mean || !S.rolling_variance)))
        return fail("missing parameter arrays", l, nm);
      const size_t need = (size_t)S.filters * c * S.size * S.size;
      if (S.n_weights != need) {
        std::string msg = "the weights hold " + std::to_string(S.n_weights) + " floats, the layer needs " + std::to_string(need);
        return fail(msg.c_str(), l, nm);
      }
      L.filters = S.filters; L.size = S.size; L.stride = S.stride; L.pad = S.pad;
      L.bn = S.batch_normalize ? 1 : 0; L.act = S.activation;
      oc = S.filters;
      oh = (h + 2 * S.pad - S.size) / S.stride + 1;
      ow = (w + 2 * S.pad - S.size) / S.stride + 1;
    } else if (S.type == B2F_DN_MAXPOOL) {
      if (S.size <= 0 || S.stride <= 0 || S.pad < 0) return fail("bad size, stride or pad", l, nm);
      L.size = S.size; L.stride = S.stride; L.pad = S.pad;
      oh = (h + 2 * S.pad) / S.stride;
      ow = (w + 2 * S.pad) / S.stride;
    } else if (S.type == B2F_DN_AVGPOOL) {
      oh = ow = 1;
    } else if (S.type == B2F_DN_SOFTMAX) {
      if (S.groups != 1 || S.tree) return fail("only groups=1 without a tree is supported", l, nm);
      L.temperature = S.temperature;
    } else if (S.type == B2F_DN_REGION) {
      if (S.tree) return fail("softmax trees are not supported", l, nm);
      if (S.coords != 4 || S.classes <= 0 || S.num <= 0 || !S.anchors) return fail("needs coords=4, classes, num and anchors", l, nm);
      if ((long long)c * h * w != (long long)w * h * S.num * (S.classes + S.coords + 1))
        return fail("its input does not hold num * (classes + coords + 1) planes", l, nm);
      L.classes = S.classes; L.coords = S.coords; L.num = S.num; L.softmax = S.softmax;
      L.anchors.assign(S.anchors, S.anchors + 2 * S.num);
      m->region = l;
      m->dims[0] = w * h * S.num;
      m->dims[1] = S.classes;
    }
    if (oh <= 0 || ow <= 0) return fail("no output at the network size", l, nm);
    if (S.type != B2F_DN_COST) m->last = l;
    c = oc; h = oh; w = ow;
  }
  if (m->n_gpu == 0) return fail("the network has no convolutional or pooling layer", 0, layers[0].name);
  m->dims[2] = c * h * w;
  // host image of the device block: the u8 table, then per conv layer weights [Kpad][Mpad], mean, scale, bias, den
  std::vector<char> img;
  auto put = [&](const void *p, size_t bytes) { const size_t o = img.size(); img.resize(align256(o + bytes), 0); if (p) std::memcpy(img.data() + o, p, bytes); return o; };
  float lut[256];
  for (int i = 0; i < 256; i++) lut[i] = (float)i / 255.;
  const size_t o_lut = put(lut, sizeof(lut));
  c = 3;
  for (int l = 0; l < n_layers; l++) {
    const b2f_darknet_layer &S = layers[l];
    DnLayer &L = m->L[l];
    if (S.type == B2F_DN_CONV) {
      L.K = c * S.size * S.size;
      L.Kpad = (L.K + DN_BK - 1) / DN_BK * DN_BK;
      L.Mpad = (S.filters + DN_MALIGN - 1) / DN_MALIGN * DN_MALIGN;
      std::vector<float> wt((size_t)L.Kpad * L.Mpad, 0.f);
      for (int f = 0; f < S.filters; f++)
        for (int k = 0; k < L.K; k++) wt[(size_t)k * L.Mpad + f] = S.weights[(size_t)f * L.K + k];
      L.o_wt = put(wt.data(), wt.size() * 4);
      L.o_bias = put(S.biases, (size_t)S.filters * 4);
      if (L.bn) {
        std::vector<double> den(S.filters);
        for (int f = 0; f < S.filters; f++) den[f] = std::sqrt((double)S.rolling_variance[f]) + .000001f;
        L.o_mean = put(S.rolling_mean, (size_t)S.filters * 4);
        L.o_scale = put(S.scales, (size_t)S.filters * 4);
        L.o_den = put(den.data(), den.size() * 8);
      }
      c = S.filters;
    }
  }
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e == cudaSuccess) e = cudaMalloc(&m->mem, img.size());
  if (e == cudaSuccess) e = cudaMemcpy(m->mem, img.data(), img.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (m->mem) cudaFree(m->mem);
    delete m;
    set_error("%s: %s", who, cudaGetErrorString(e));
    return B2F_ECUDA;
  }
  char *base = static_cast<char *>(m->mem);
  m->lut = reinterpret_cast<const float *>(base + o_lut);
  for (DnLayer &L : m->L) {
    if (L.type != B2F_DN_CONV) continue;
    L.wt = reinterpret_cast<const float *>(base + L.o_wt);
    L.bias = reinterpret_cast<const float *>(base + L.o_bias);
    if (L.bn) {
      L.mean = reinterpret_cast<const float *>(base + L.o_mean);
      L.scale = reinterpret_cast<const float *>(base + L.o_scale);
      L.den = reinterpret_cast<const double *>(base + L.o_den);
    }
  }
  *model = m;
  return B2F_OK;
}

void b2f_darknet_model_free(b2f_darknet_model *model) {
  if (!model) return;
  cudaSetDevice(model->device);
  cudaFree(model->mem);
  delete model;
}

int b2f_darknet_model_dims(const b2f_darknet_model *model, int *dims) {
  if (!model || !dims) { set_error("b2f_darknet_model_dims: bad argument"); return B2F_EINVAL; }
  std::copy(model->dims, model->dims + 3, dims);
  return B2F_OK;
}

int b2f_darknet_detect_batch_rgb(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *frames, int n_frames, int width,
                                 int height, float thresh, float hier_thresh, float *probs, float *boxes, int *count) {
  const char *who = "b2f_darknet_detect_batch_rgb";
  (void)hier_thresh;
  if (!ctx || !frames || !probs || !boxes || !count) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  int rc = dn_check(who, model, n_frames, width, height);
  if (rc == B2F_OK) rc = dn_check_detect(who, model);
  DnGeom g;
  if (rc == B2F_OK) rc = dn_geom(who, model, 0, width, height, g);
  if (rc != B2F_OK) return rc;
  const size_t per = (size_t)model->dims[0];
  const size_t np = (size_t)model->dims[1] + 1;
  return dn_batch(who, ctx, g, frames, n_frames, width, height, [&](const uint8_t *d, int f0, int nf, cudaStream_t st) {
    return dn_detect_frames(ctx, model, g, d, nf, width, height,
                            DnDetectOut{thresh, probs + f0 * per * np, boxes + f0 * per * 4, count + f0}, st);
  });
}

int b2f_darknet_detect_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                           int height, float thresh, float hier_thresh, float *probs, float *boxes, int *count, void *stream) {
  const char *who = "b2f_darknet_detect_dev";
  (void)hier_thresh;
  if (!ctx || !d_frames || !probs || !boxes || !count) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  int rc = dn_check(who, model, n_frames, width, height);
  if (rc == B2F_OK) rc = dn_check_detect(who, model);
  DnGeom g;
  if (rc == B2F_OK) rc = dn_geom(who, model, 0, width, height, g);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, dn_scratch_bytes(g, n_frames))) != B2F_OK) return rc;
  return dn_detect_frames(ctx, model, g, d_frames, n_frames, width, height, DnDetectOut{thresh, probs, boxes, count}, st);
}

int b2f_darknet_classify_batch_rgb(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *frames, int n_frames, int width,
                                   int height, int resize, int top, int *index, double *prob) {
  const char *who = "b2f_darknet_classify_batch_rgb";
  if (!ctx || !frames || !index || !prob) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  int rc = dn_check(who, model, n_frames, width, height);
  if (rc == B2F_OK) rc = dn_check_classify(who, model, top);
  DnGeom g;
  if (rc == B2F_OK) rc = dn_geom(who, model, resize ? 1 : 2, width, height, g);
  if (rc != B2F_OK) return rc;
  return dn_batch(who, ctx, g, frames, n_frames, width, height, [&](const uint8_t *d, int f0, int nf, cudaStream_t st) {
    return dn_classify_frames(ctx, model, g, d, nf, width, height,
                              DnClassifyOut{resize, top, index + (size_t)f0 * top, prob + (size_t)f0 * top}, st);
  });
}

int b2f_darknet_classify_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                             int height, int resize, int top, int *index, double *prob, void *stream) {
  const char *who = "b2f_darknet_classify_dev";
  if (!ctx || !d_frames || !index || !prob) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  int rc = dn_check(who, model, n_frames, width, height);
  if (rc == B2F_OK) rc = dn_check_classify(who, model, top);
  DnGeom g;
  if (rc == B2F_OK) rc = dn_geom(who, model, resize ? 1 : 2, width, height, g);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, dn_scratch_bytes(g, n_frames))) != B2F_OK) return rc;
  return dn_classify_frames(ctx, model, g, d_frames, n_frames, width, height, DnClassifyOut{resize, top, index, prob}, st);
}

int b2f_darknet_layer_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                          int height, int mode, int layer, float *out, size_t out_len, int *dims, void *stream) {
  const char *who = "b2f_darknet_layer_dev";
  if (!ctx || !d_frames || !dims || mode < 0 || mode > 2) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  int rc = dn_check(who, model, n_frames, width, height);
  if (rc != B2F_OK) return rc;
  if (layer < -1 || layer >= (int)model->L.size() || (layer >= 0 && model->L[layer].type == B2F_DN_COST)) {
    set_error("%s: layer %d is not a layer with an output", who, layer);
    return B2F_EINVAL;
  }
  DnGeom g;
  if ((rc = dn_geom(who, model, mode, width, height, g)) != B2F_OK) return rc;
  if (layer < 0) { dims[0] = 3; dims[1] = g.RH; dims[2] = g.RW; }
  else if (layer < model->n_gpu) { dims[0] = g.oc[layer]; dims[1] = g.oh[layer]; dims[2] = g.ow[layer]; }
  else { dims[0] = g.oc[model->n_gpu - 1] * g.oh[model->n_gpu - 1] * g.ow[model->n_gpu - 1]; dims[1] = dims[2] = 1; }
  if (!out) return B2F_OK;
  const size_t per = (size_t)dims[0] * dims[1] * dims[2];
  if (out_len < per * n_frames) { set_error("%s: out holds %zu floats, %zu needed", who, out_len, per * n_frames); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, dn_scratch_bytes(g, n_frames))) != B2F_OK) return rc;
  const float *d_out = nullptr;
  if ((rc = dn_forward(ctx, model, g, d_frames, n_frames, width, height, std::min(layer, model->n_gpu - 1), &d_out, st)) != B2F_OK) return rc;
  if (layer < model->n_gpu) {
    B2F_CUDA(cudaMemcpyAsync(out, d_out, per * n_frames * 4, cudaMemcpyDeviceToHost, st));
    B2F_CUDA(cudaStreamSynchronize(st));
    return B2F_OK;
  }
  std::vector<float> x((size_t)n_frames * per), y;
  B2F_CUDA(cudaMemcpyAsync(x.data(), d_out, x.size() * 4, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  for (int f = 0; f < n_frames; f++) {
    dn_host_layers(model, g, x.data() + (size_t)f * per, layer, y);
    std::copy(y.begin(), y.end(), out + (size_t)f * per);
  }
  return B2F_OK;
}

}  // extern "C"
