// facedetect.cu — the CNN face detector of image.libfacedetection (detect_faces -> facedetect_cnn -> objectdetect_cnn,
// facedetectcnn-model.cpp:103-437), bit-identical to the reference built with gcc -O2 on x86-64.
// The network is an int8 CNN: u8 activations times s8 weights summed in int32, so any summation order gives the
// reference's int32 planes; only the per-layer scalars, the requantisation and the detection tail involve floats.
//   fd_conv0_kernel          layer 0 (3x3, stride 2, pad 1 over RGB) straight from the interleaved frame, integer MACs;
//                            the reference's 27-channel im2col blob never exists.
//   fd_conv_mma_kernel<NT,KS> every other layer (16..256 input channels): implicit GEMM on the tensor cores with
//                            mma.sync.m16n8k32.s32.u8.s8.s32.  M = pixels, N = output channels, K = tap * C + c over NHWC
//                            u8 activations.  The epilogue adds in.bias * f.bias (wrapping, as the reference's int
//                            multiply does), and for ReLU layers clamps at 0 and folds the frame's maximum into one
//                            atomicMax per warp.  Fragments are loaded straight from global memory (L1/L2 resident).
//   fd_scalars_kernel        one thread per frame: nMax -> s = 255/nMax, scale and bias of the layer, with x86 conversions.
//   fd_requant_kernel        int32 -> u8 = (unsigned char)(v * s + 0.499f); fd_requant_pool_kernel does the same on the
//                            2x2 maximum (requantisation is monotone non-decreasing, so pool(requant) = requant(pool)).
//   fd_cand_kernel           every prior whose conf ints satisfy i1 > i0 (all priors of a head with a degenerate scale),
//                            with its 2 conf and 14 loc ints; the detection tail runs on the host on these records only.
#include "common.cuh"
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <vector>

namespace b2f {

__global__ void narrow_i32_to_u8_kernel(const int *__restrict__ src, unsigned char *__restrict__ dst, size_t n);   // ingest.cu

constexpr int FD_NL = 24, FD_NRELU = 16, FD_REC = 17;
constexpr size_t FD_CHUNK_SCRATCH = (size_t)2 << 30;      // scratch bytes one chunk of a batch may use
struct FdShape { int k, c, n; };
// facedetectcnn-model.cpp:132-310 with the shapes of facedetectcnn-int8data.cpp's table
static const FdShape FD_SHAPE[FD_NL] = {
    {3, 3, 32}, {1, 32, 16}, {3, 16, 32}, {1, 32, 32}, {3, 32, 64}, {1, 64, 32}, {3, 32, 64}, {3, 64, 128},
    {1, 128, 64}, {3, 64, 128}, {3, 128, 256}, {1, 256, 128}, {3, 128, 256}, {3, 256, 256}, {1, 256, 256}, {3, 256, 256},
    {3, 64, 42}, {3, 64, 6}, {3, 128, 28}, {3, 128, 4}, {3, 256, 28}, {3, 256, 4}, {3, 256, 42}, {3, 256, 6}};
static const bool FD_POOL_AFTER[FD_NRELU] = {0, 1, 0, 1, 0, 0, 1, 0, 0, 1, 0, 0, 1, 0, 0, 0};
static const int FD_HEAD_SRC[4] = {6, 9, 12, 15}, FD_HEAD_NS[4] = {3, 2, 2, 3}, FD_HEAD_STEP[4] = {8, 16, 32, 64};
static const float FD_HEAD_SIZE[4][3] = {{10, 16, 24}, {32, 48, 0}, {64, 96, 0}, {128, 192, 256}};

struct FdState {              // per frame: the scalars of each ReLU layer's output blob
  float scale[FD_NRELU];
  int bias[FD_NRELU];
  float s[FD_NRELU];          // 255 / nMax
};

struct FdGemm {               // one tensor-core convolution: weights [Npad][Kpad] with K = tap * C + c, zero padded
  int8_t *w;
  int32_t *bias;              // [Npad]
  int ks, C, N, Npad, Kpad, nt;
};

}  // namespace b2f

struct b2f_facedet_model {
  int device;
  float fscale[b2f::FD_NL];
  void *mem;                  // one device block: layer 0's weights and bias, then every FdGemm's
  int8_t *w0;                 // [32][27], k = (ky * 3 + kx) * 3 + colour (the reference's blob2vector order)
  int32_t *b0;
  b2f::FdGemm g[19];          // L1..L15, then the four heads with loc and conf fused (loc channels first)
};

namespace b2f {

// (int)f as gcc compiles it on x86-64 (cvttss2si): NaN and out-of-range values give INT_MIN
__host__ __device__ __forceinline__ int fd_cvtt(float f) {
  return (f != f || f >= 2147483648.0f || f < -2147483648.0f) ? INT_MIN : (int)f;
}

__device__ __forceinline__ unsigned char fd_requant(int v, float s) {
  return (unsigned char)fd_cvtt(__fadd_rn(__fmul_rn(__int2float_rn(v), s), 0.499f));
}

__device__ __forceinline__ void fd_mma(int *c, const uint32_t *a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

__device__ __forceinline__ void fd_fold_max(int v, int *slot) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = max(v, __shfl_xor_sync(0xffffffffu, v, o));
  if ((threadIdx.x & 31) == 0 && v > 0) atomicMax(slot, v);
}

// in_bias of a layer: the output bias of its source ReLU layer, or 1 for the image (setDataFrom3x3S2P1to1x1S1P0FromImage)
__device__ __forceinline__ int fd_in_bias(const FdState *st, int f, int src) { return src < 0 ? 1 : st[f].bias[src]; }

// Layer 0: one thread per output pixel, all 32 channels.  out int32 [f][H0*W0][32] after ReLU.
__global__ void __launch_bounds__(128) fd_conv0_kernel(const uint8_t *__restrict__ rgb, int W, int H, int W0, int H0,
                                                       const int8_t *__restrict__ w, const int32_t *__restrict__ bias,
                                                       int32_t *__restrict__ out, int *__restrict__ lmax) {
  __shared__ int sw[32 * 27], sb[32];
  for (int i = threadIdx.x; i < 32 * 27; i += 128) sw[i] = w[i];
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  __syncthreads();
  const int f = blockIdx.y;
  const int p = blockIdx.x * 128 + threadIdx.x;
  const int M0 = W0 * H0;
  int vmax = 0;
  if (p < M0) {
    const int x0 = p % W0, y0 = p / W0;
    const uint8_t *img = rgb + (size_t)f * W * H * 3;
    int v[27];
#pragma unroll
    for (int t = 0; t < 9; t++) {
      const int sy = 2 * y0 + t / 3 - 1, sx = 2 * x0 + t % 3 - 1;
      const bool ok = sy >= 0 && sy < H && sx >= 0 && sx < W;
#pragma unroll
      for (int c = 0; c < 3; c++) v[t * 3 + c] = ok ? img[((size_t)sy * W + sx) * 3 + c] : 0;
    }
    int32_t *o = out + ((size_t)f * M0 + p) * 32;
#pragma unroll 4
    for (int n = 0; n < 32; n++) {
      int s = 0;
#pragma unroll
      for (int k = 0; k < 27; k++) s += v[k] * sw[n * 27 + k];
      s = max((int)((unsigned)s + (unsigned)sb[n]), 0);         // + in.bias (1) * f.bias, then ReLU
      vmax = max(vmax, s);
      o[n] = s;
    }
  }
  fd_fold_max(vmax, lmax + f * FD_NRELU);
}

struct FdConvArgs {
  const uint8_t *in;          // [f][H][W][C] u8
  const int8_t *w;            // [Npad][Kpad]
  const int32_t *bias;        // [Npad]
  int32_t *out;               // [f][H*W][N]
  const FdState *st;
  int *lmax;                  // &layer_max[0][l] for a ReLU layer (frame stride FD_NRELU), nullptr for a head
  int H, W, C, cshift, Kpad, N, src;
};

// Implicit GEMM, one warp = 32 pixels x 8*NT channels, four warps per CTA.  mma m16n8k32 fragments (PTX ISA, integer
// m16n8k32): A reg r of thread (g = lane/4, t = lane%4) holds row g + 8*(r&1), columns 16*(r>>1) + 4t..4t+3; B reg r holds
// column g, rows 16r + 4t..4t+3; C holds rows g, g+8 and columns 2t, 2t+1.  C is a multiple of 4, so each 4-column group
// is 4 consecutive channels of one tap: one 32-bit load.
template <int NT, int KS>
__global__ void __launch_bounds__(128) fd_conv_mma_kernel(FdConvArgs a) {
  const int f = blockIdx.z, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int H = a.H, W = a.W, C = a.C, M = H * W;
  const int m0 = (blockIdx.x * 4 + warp) * 32, n0 = blockIdx.y * 8 * NT;
  const uint8_t *in = a.in + (size_t)f * M * C;
  int py[4], px[4];
#pragma unroll
  for (int r = 0; r < 4; r++) {
    const int m = m0 + g + 8 * r;
    py[r] = m < M ? m / W : -0x40000000;                 // a row no tap reaches: the pixel loads zeros
    px[r] = m < M ? m % W : 0;
  }
  int acc[2][NT][4];
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < NT; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) acc[i][j][e] = 0;
  const int8_t *wrow = a.w + (size_t)(n0 + g) * a.Kpad + t * 4;
  for (int kb = 0; kb < a.Kpad; kb += 32) {
    uint32_t A[2][4];
#pragma unroll
    for (int h = 0; h < 2; h++) {
      const int k = kb + h * 16 + t * 4;
      const int tap = k >> a.cshift, c = k & (C - 1);
      const int dy = KS == 3 ? tap / 3 - 1 : 0, dx = KS == 3 ? tap % 3 - 1 : 0;
      const bool tv = KS == 3 ? tap < 9 : true;
#pragma unroll
      for (int r = 0; r < 4; r++) {
        const int yy = py[r] + dy, xx = px[r] + dx;
        uint32_t v = 0;
        if (tv && yy >= 0 && yy < H && xx >= 0 && xx < W)
          v = __ldg(reinterpret_cast<const uint32_t *>(in + ((size_t)yy * W + xx) * C + c));
        A[r >> 1][(r & 1) + 2 * h] = v;
      }
    }
#pragma unroll
    for (int j = 0; j < NT; j++) {
      const int8_t *wp = wrow + (size_t)j * 8 * a.Kpad + kb;
      const uint32_t b0 = __ldg(reinterpret_cast<const uint32_t *>(wp)), b1 = __ldg(reinterpret_cast<const uint32_t *>(wp + 16));
      fd_mma(acc[0][j], A[0], b0, b1);
      fd_mma(acc[1][j], A[1], b0, b1);
    }
  }
  const unsigned ib = (unsigned)fd_in_bias(a.st, f, a.src);
  int32_t *out = a.out + (size_t)f * M * a.N;
  int vmax = 0;
#pragma unroll
  for (int i = 0; i < 2; i++)
#pragma unroll
    for (int j = 0; j < NT; j++)
#pragma unroll
      for (int e = 0; e < 4; e++) {
        const int m = m0 + i * 16 + g + (e >> 1) * 8, n = n0 + j * 8 + t * 2 + (e & 1);
        if (m < M && n < a.N) {
          int v = (int)((unsigned)acc[i][j][e] + ib * (unsigned)__ldg(a.bias + n));
          if (a.lmax) { v = max(v, 0); vmax = max(vmax, v); }
          out[(size_t)m * a.N + n] = v;
        }
      }
  if (a.lmax) fd_fold_max(vmax, a.lmax + f * FD_NRELU);
}

// convolution() and convolution_relu() scalars (facedetectcnn.cpp:353-354, 450-453) for ReLU layer l of every frame
__global__ void fd_scalars_kernel(FdState *st, const int *__restrict__ lmax, int l, float fscale, int n) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const float in_scale = l == 0 ? 1.0f : st[f].scale[l - 1];
  const float cs = __fmul_rn(in_scale, fscale);
  const int cb = fd_cvtt(roundf(cs));
  const float s = __fdiv_rn(255.0f, __int2float_rn(lmax[f * FD_NRELU + l]));
  st[f].s[l] = s;
  st[f].scale[l] = __fmul_rn(cs, s);
  st[f].bias[l] = fd_cvtt(roundf(__fmul_rn(__int2float_rn(cb), s)));
}

// int32 [f][M][N] -> u8 [f][M][N], four channels per thread (N is a multiple of 4)
__global__ void __launch_bounds__(256) fd_requant_kernel(const int32_t *__restrict__ in, uint8_t *__restrict__ out, size_t quads,
                                                         const FdState *st, int l) {
  const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x;
  const int f = blockIdx.y;
  if (q >= quads) return;
  const float s = st[f].s[l];
  const int4 v = __ldg(reinterpret_cast<const int4 *>(in) + (size_t)f * quads + q);
  reinterpret_cast<uint32_t *>(out)[(size_t)f * quads + q] =
      fd_requant(v.x, s) | (fd_requant(v.y, s) << 8) | (fd_requant(v.z, s) << 16) | ((uint32_t)fd_requant(v.w, s) << 24);
}

// int32 [f][H][W][N] -> u8 [f][H/2][W/2][N]: maxpooling2x2S2 (an odd last row or column is dropped) of the requantised plane
__global__ void __launch_bounds__(256) fd_requant_pool_kernel(const int32_t *__restrict__ in, uint8_t *__restrict__ out, int W, int H,
                                                              int N, const FdState *st, int l) {
  const int Wp = W / 2, Hp = H / 2, nq = N / 4;
  const size_t q = (size_t)blockIdx.x * 256 + threadIdx.x, total = (size_t)Wp * Hp * nq;
  const int f = blockIdx.y;
  if (q >= total) return;
  const int c4 = (int)(q % nq);
  const size_t p = q / nq;
  const int x = (int)(p % Wp), y = (int)(p / Wp);
  const int4 *src = reinterpret_cast<const int4 *>(in + (size_t)f * W * H * N);
  int4 m = __ldg(src + ((size_t)(2 * y) * W + 2 * x) * nq + c4);
#pragma unroll
  for (int d = 1; d < 4; d++) {
    const int4 v = __ldg(src + ((size_t)(2 * y + (d >> 1)) * W + 2 * x + (d & 1)) * nq + c4);
    m.x = max(m.x, v.x); m.y = max(m.y, v.y); m.z = max(m.z, v.z); m.w = max(m.w, v.w);
  }
  const float s = st[f].s[l];
  reinterpret_cast<uint32_t *>(out)[(size_t)f * total + q] =
      fd_requant(m.x, s) | (fd_requant(m.y, s) << 8) | (fd_requant(m.z, s) << 16) | ((uint32_t)fd_requant(m.w, s) << 24);
}

// Candidate records of one head: plane [f][M][N] with the 14*ns loc channels first, then the 2*ns conf channels.
// For 1/scale positive and finite, i1 <= i0 gives c1 <= c0 after convertInt2Float, and the softmax then gives at most 0.5,
// which fails `> 0.5`: such a prior can never be kept.  For any other 1/scale every prior is sent.
__global__ void __launch_bounds__(256) fd_cand_kernel(const int32_t *__restrict__ plane, int M, int N, int ns, const FdState *st,
                                                      int src, float fscale_conf, int base, int *count, int32_t *rec, int cap) {
  const int i = blockIdx.x * 256 + threadIdx.x, f = blockIdx.y;
  if (i >= M * ns) return;
  const int j = i % ns;
  const int32_t *p = plane + ((size_t)f * M + i / ns) * N;
  const int i0 = p[14 * ns + 2 * j], i1 = p[14 * ns + 2 * j + 1];
  const float inv = __fdiv_rn(1.0f, __fmul_rn(st[f].scale[src], fscale_conf));
  const bool all = !(inv > 0.0f && inv <= FLT_MAX);
  if (!all && i1 <= i0) return;
  const int pos = atomicAdd(count + f, 1);
  if (pos >= cap) return;
  int32_t *r = rec + ((size_t)f * cap + pos) * FD_REC;
  r[0] = base + i; r[1] = i0; r[2] = i1;
#pragma unroll
  for (int k = 0; k < 14; k++) r[3 + k] = p[14 * j + k];
}

// ------------------------------------------------------------------------------------------------ geometry, scratch --
struct FdGeom {
  int W, H;
  int lw[FD_NRELU], lh[FD_NRELU];  // output size of each ReLU layer
  int n_run;                       // ReLU layers the reference runs: a pool whose output would be empty stops the chain
  int head_off[5];                 // first prior index of each head; head_off[4] = priors per frame
};

static FdGeom fd_geom(int W, int H) {
  FdGeom g{};
  g.W = W; g.H = H;
  if (W < 1 || H < 1) return g;
  int w = (W + 1) / 2, h = (H + 1) / 2;            // convolution(): 3x3 stride 2 pad 1
  for (int l = 0; l < FD_NRELU; l++) {
    g.lw[l] = w; g.lh[l] = h; g.n_run = l + 1;
    if (FD_POOL_AFTER[l]) {                        // maxpooling2x2S2 (facedetectcnn.cpp:479-487)
      w = (int)std::ceil((w - 3.0f) / 2) + 1;
      h = (int)std::ceil((h - 3.0f) / 2) + 1;
      if (w < 1 || h < 1) break;
    }
  }
  for (int hd = 0; hd < 4; hd++) {
    const int s = FD_HEAD_SRC[hd];
    g.head_off[hd + 1] = g.head_off[hd] + (g.n_run == FD_NRELU ? g.lw[s] * g.lh[s] * FD_HEAD_NS[hd] : 0);
  }
  return g;
}

static bool fd_keep_unpooled(int l) { return !FD_POOL_AFTER[l] || l == 6 || l == 9 || l == 12; }

// Device scratch of n frames of W x H: the int32 plane of the largest layer, every u8 activation, the records and the
// per-frame slots.  Used to reserve the arena and to cut batches into chunks.
size_t facedet_scratch_bytes(int W, int H, int n) {
  const FdGeom g = fd_geom(W, H);
  size_t plane = 0, act = 0;
  for (int l = 0; l < g.n_run; l++) {
    const size_t M = (size_t)g.lw[l] * g.lh[l];
    plane = std::max(plane, M * FD_SHAPE[l].n * 4);
    if (fd_keep_unpooled(l)) act += align256((size_t)n * M * FD_SHAPE[l].n);
    if (FD_POOL_AFTER[l] && l + 1 < g.n_run) act += align256((size_t)n * (g.lw[l] / 2) * (g.lh[l] / 2) * FD_SHAPE[l].n);
  }
  if (g.n_run == FD_NRELU)
    for (int hd = 0; hd < 4; hd++) {
      const int s = FD_HEAD_SRC[hd];
      plane = std::max(plane, (size_t)g.lw[s] * g.lh[s] * (FD_SHAPE[16 + 2 * hd].n + FD_SHAPE[17 + 2 * hd].n) * 4);
    }
  return align256(plane * n) + act + align256((size_t)n * FD_NRELU * 4) + align256((size_t)n * sizeof(FdState)) +
         align256((size_t)n * 4) + align256((size_t)n * std::max(g.head_off[4], 1) * FD_REC * 4);
}

// What one launch sequence leaves on the host for the tail
struct FdHostOut {
  std::vector<int> lmax;        // [n][16]
  std::vector<FdState> st;      // [n]
  std::vector<int> count;       // [n]
  std::vector<int32_t> rec;     // [n][cap][17], the first count[f] of each frame valid
  int cap = 0;
};

static int fd_launch_gemm(b2f_ctx *ctx, const FdGemm &G, const FdConvArgs &a, int n, cudaStream_t st) {
  const dim3 grid(ceil_div(a.H * a.W, 128), G.Npad / (8 * G.nt), n);
  if (G.nt == 4) {
    if (G.ks == 3) fd_conv_mma_kernel<4, 3><<<grid, 128, 0, st>>>(a);
    else fd_conv_mma_kernel<4, 1><<<grid, 128, 0, st>>>(a);
  } else {
    if (G.ks == 3) fd_conv_mma_kernel<2, 3><<<grid, 128, 0, st>>>(a);
    else fd_conv_mma_kernel<2, 1><<<grid, 128, 0, st>>>(a);
  }
  B2F_LAUNCH_CHECK(ctx);
  return B2F_OK;
}

static int fd_log2(int c) { int s = 0; while ((1 << s) < c) s++; return s; }

// n frames [n][H][W][3] u8 in HBM -> the per-frame maxima, scalars and candidate records on the host.  The arena is
// reserved by the caller for facedet_scratch_bytes(W, H, n); one launch sequence, no host round trip between layers.
static int fd_device(b2f_ctx *ctx, const b2f_facedet_model *m, const uint8_t *d_rgb, int n, int W, int H, FdHostOut &ho,
                     cudaStream_t st) {
  const FdGeom g = fd_geom(W, H);
  const size_t mark = ctx->arena.off;
  size_t plane_elems = 0;
  for (int l = 0; l < g.n_run; l++) plane_elems = std::max(plane_elems, (size_t)g.lw[l] * g.lh[l] * FD_SHAPE[l].n);
  if (g.n_run == FD_NRELU)
    for (int hd = 0; hd < 4; hd++)
      plane_elems = std::max(plane_elems, (size_t)g.lw[FD_HEAD_SRC[hd]] * g.lh[FD_HEAD_SRC[hd]] * m->g[15 + hd].N);
  int32_t *plane = ctx->arena.get<int32_t>(plane_elems * n);
  uint8_t *act[FD_NRELU] = {}, *pooled[FD_NRELU] = {};
  for (int l = 0; l < g.n_run; l++) {
    const size_t M = (size_t)g.lw[l] * g.lh[l];
    if (fd_keep_unpooled(l)) act[l] = ctx->arena.get<uint8_t>((size_t)n * M * FD_SHAPE[l].n);
    if (FD_POOL_AFTER[l] && l + 1 < g.n_run) pooled[l] = ctx->arena.get<uint8_t>((size_t)n * (g.lw[l] / 2) * (g.lh[l] / 2) * FD_SHAPE[l].n);
  }
  int *lmax = ctx->arena.get<int>((size_t)n * FD_NRELU);
  FdState *dst = ctx->arena.get<FdState>(n);
  int *count = ctx->arena.get<int>(n);
  const int cap = std::max(g.head_off[4], 1);      // every prior fits: the list cannot overflow
  int32_t *rec = ctx->arena.get<int32_t>((size_t)n * cap * FD_REC);
  B2F_ARENA_CHECK(ctx);
  ctx->arena.off = mark;
  B2F_CUDA(cudaMemsetAsync(lmax, 0, sizeof(int) * n * FD_NRELU, st));
  B2F_CUDA(cudaMemsetAsync(count, 0, sizeof(int) * n, st));
  B2F_CUDA(cudaMemsetAsync(dst, 0, sizeof(FdState) * n, st));
  int rc;
  for (int l = 0; l < g.n_run; l++) {
    const int M = g.lw[l] * g.lh[l], N = FD_SHAPE[l].n;
    if (l == 0) {
      fd_conv0_kernel<<<dim3(ceil_div(M, 128), n), 128, 0, st>>>(d_rgb, W, H, g.lw[0], g.lh[0], m->w0, m->b0, plane, lmax);
      B2F_LAUNCH_CHECK(ctx);
    } else {
      const int pl = l - 1;
      const uint8_t *in = FD_POOL_AFTER[pl] ? pooled[pl] : act[pl];
      const FdGemm &G = m->g[l - 1];
      FdConvArgs a{in, G.w, G.bias, plane, dst, lmax + l, g.lh[l], g.lw[l], G.C, fd_log2(G.C), G.Kpad, N, l - 1};
      if ((rc = fd_launch_gemm(ctx, G, a, n, st)) != B2F_OK) return rc;
    }
    fd_scalars_kernel<<<ceil_div(n, 128), 128, 0, st>>>(dst, lmax, l, m->fscale[l], n);
    B2F_LAUNCH_CHECK(ctx);
    if (act[l]) {
      const size_t quads = (size_t)M * N / 4;
      fd_requant_kernel<<<dim3((unsigned)((quads + 255) / 256), n), 256, 0, st>>>(plane, act[l], quads, dst, l);
      B2F_LAUNCH_CHECK(ctx);
    }
    if (pooled[l]) {
      const size_t quads = (size_t)(g.lw[l] / 2) * (g.lh[l] / 2) * N / 4;
      fd_requant_pool_kernel<<<dim3((unsigned)((quads + 255) / 256), n), 256, 0, st>>>(plane, pooled[l], g.lw[l], g.lh[l], N, dst, l);
      B2F_LAUNCH_CHECK(ctx);
    }
  }
  if (g.n_run == FD_NRELU)
    for (int hd = 0; hd < 4; hd++) {
      const int s = FD_HEAD_SRC[hd], M = g.lw[s] * g.lh[s];
      const FdGemm &G = m->g[15 + hd];
      FdConvArgs a{act[s], G.w, G.bias, plane, dst, nullptr, g.lh[s], g.lw[s], G.C, fd_log2(G.C), G.Kpad, G.N, s};
      if ((rc = fd_launch_gemm(ctx, G, a, n, st)) != B2F_OK) return rc;
      fd_cand_kernel<<<dim3(ceil_div(M * FD_HEAD_NS[hd], 256), n), 256, 0, st>>>(plane, M, G.N, FD_HEAD_NS[hd], dst, s,
                                                                                  m->fscale[17 + 2 * hd], g.head_off[hd], count, rec, cap);
      B2F_LAUNCH_CHECK(ctx);
    }
  ho.lmax.resize((size_t)n * FD_NRELU);
  ho.st.resize(n);
  ho.count.resize(n);
  ho.cap = cap;
  B2F_CUDA(cudaMemcpyAsync(ho.lmax.data(), lmax, sizeof(int) * n * FD_NRELU, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaMemcpyAsync(ho.st.data(), dst, sizeof(FdState) * n, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaMemcpyAsync(ho.count.data(), count, sizeof(int) * n, cudaMemcpyDeviceToHost, st));
  B2F_CUDA(cudaStreamSynchronize(st));
  size_t total = 0;
  for (int f = 0; f < n; f++) total += (size_t)std::min(ho.count[f], cap);
  ho.rec.assign(total * FD_REC, 0);
  size_t off = 0;
  for (int f = 0; f < n; f++) {                    // compact: frame f's records follow frame f-1's
    const size_t c = (size_t)std::min(ho.count[f], cap);
    if (c) B2F_CUDA(cudaMemcpyAsync(ho.rec.data() + off * FD_REC, rec + (size_t)f * cap * FD_REC, c * FD_REC * 4, cudaMemcpyDeviceToHost, st));
    off += c;
  }
  B2F_CUDA(cudaStreamSynchronize(st));
  for (int f = 0; f < n; f++)
    for (int l = g.n_run; l < FD_NRELU; l++) ho.lmax[(size_t)f * FD_NRELU + l] = -1;
  return B2F_OK;
}

// ---------------------------------------------------------------------------------------------------- host tail --
// facedetectcnn.cpp:624-951 and facedetectcnn-model.cpp:343-436 on the candidate records of one frame.  This file is
// compiled with -ffp-contract=off, and expf is the C library's, as in the reference.
struct FdBox { float xmin, ymin, xmax, ymax, lm[10]; };

#define FD_MIN(a, b) ((a) > (b) ? (b) : (a))       // facedetectcnn.h:104-110
#define FD_MAX(a, b) ((a) < (b) ? (b) : (a))

static float fd_jaccard(const FdBox &b1, const FdBox &b2) {       // IntersectBBox + JaccardOverlap (:763-803)
  float ix0, iy0, ix1, iy1;
  if (b2.xmin > b1.xmax || b2.xmax < b1.xmin || b2.ymin > b1.ymax || b2.ymax < b1.ymin) {
    ix0 = iy0 = ix1 = iy1 = 0;
  } else {
    ix0 = std::max(b1.xmin, b2.xmin); iy0 = std::max(b1.ymin, b2.ymin);
    ix1 = std::min(b1.xmax, b2.xmax); iy1 = std::min(b1.ymax, b2.ymax);
  }
  const float iw = ix1 - ix0, ih = iy1 - iy0;
  if (iw > 0 && ih > 0) {
    const float is = iw * ih;
    const float s1 = (b1.xmax - b1.xmin) * (b1.ymax - b1.ymin);
    const float s2 = (b2.xmax - b2.xmin) * (b2.ymax - b2.ymin);
    return is / (s1 + s2 - is);
  }
  return 0.f;
}

static int fd_tail(const b2f_facedet_model *m, const FdGeom &g, const FdState &st, const int32_t *rec, int nrec, int *n_faces,
                   int32_t *faces) {
  std::vector<int> order(nrec);
  for (int i = 0; i < nrec; i++) order[i] = i;
  std::sort(order.begin(), order.end(), [&](int a, int b) { return rec[(size_t)a * FD_REC] < rec[(size_t)b * FD_REC]; });
  float sl[4], sc[4];
  for (int hd = 0; hd < 4; hd++) {                 // convertInt2Float (:633): s = 1.0f / scale
    const float in_scale = st.scale[FD_HEAD_SRC[hd]];
    sl[hd] = 1.0f / (in_scale * m->fscale[16 + 2 * hd]);
    sc[hd] = 1.0f / (in_scale * m->fscale[17 + 2 * hd]);
  }
  const float var[4] = {0.1f, 0.1f, 0.2f, 0.2f};
  std::vector<std::pair<float, FdBox>> cand, kept;
  for (int oi = 0; oi < nrec; oi++) {
    const int32_t *r = rec + (size_t)order[oi] * FD_REC;
    const int idx = r[0];
    int hd = 0;
    while (idx >= g.head_off[hd + 1]) hd++;
    const int ns = FD_HEAD_NS[hd], q = idx - g.head_off[hd], j = q % ns, p = q / ns;
    const int fw = g.lw[FD_HEAD_SRC[hd]], col = p % fw, row = p / fw;
    // softmax1vector2class (:716-728)
    float v1 = r[1] * sc[hd], v2 = r[2] * sc[hd];
    float vm = FD_MAX(v1, v2);
    v1 -= vm; v2 -= vm;
    v1 = expf(v1); v2 = expf(v2);
    vm = v1 + v2;
    const float conf = v2 / vm;
    if (!(conf > 0.5f)) continue;
    // priorbox (:674-688)
    const float step = (float)FD_HEAD_STEP[hd], size = FD_HEAD_SIZE[hd][j];
    const float cx = (col + 0.5f) * step, cy = (row + 0.5f) * step;
    float x1 = (cx - size / 2.f) / g.W, y1 = (cy - size / 2.f) / g.H;
    float x2 = (cx + size / 2.f) / g.W, y2 = (cy + size / 2.f) / g.H;
    // detection_output's decoding (:841-887)
    float loc[14];
    for (int k = 0; k < 14; k++) loc[k] = r[3 + k] * sl[hd];
    const float pw = x2 - x1, ph = y2 - y1, pcx = (x1 + x2) / 2, pcy = (y1 + y2) / 2;
    const float bcx = var[0] * loc[0] * pw + pcx, bcy = var[1] * loc[1] * ph + pcy;
    const float bw = expf(var[2] * loc[2]) * pw, bh = expf(var[3] * loc[3]) * ph;
    x1 = bcx - bw / 2.f; y1 = bcy - bh / 2.f; x2 = bcx + bw / 2.f; y2 = bcy + bh / 2.f;
    FdBox bb;
    bb.xmin = FD_MAX(0, x1); bb.ymin = FD_MAX(0, y1); bb.xmax = FD_MIN(1.f, x2); bb.ymax = FD_MIN(1.f, y2);
    for (int i = 0; i < 5; i++) {
      bb.lm[i * 2] = var[0] * loc[4 + i * 2] * pw + pcx;
      bb.lm[i * 2 + 1] = var[1] * loc[4 + i * 2 + 1] * ph + pcy;
    }
    cand.push_back(std::make_pair(conf, bb));
  }
  std::stable_sort(cand.begin(), cand.end(), [](const std::pair<float, FdBox> &a, const std::pair<float, FdBox> &b) { return a.first > b.first; });
  if (cand.size() > 1000) cand.resize(1000);       // top_k
  for (size_t i = 0; i < cand.size(); i++) {       // NMS (:902-922)
    bool keep = true;
    for (size_t k = 0; k < kept.size() && keep; k++) keep = fd_jaccard(cand[i].second, kept[k].second) <= 0.3f;
    if (keep) kept.push_back(cand[i]);
  }
  if (kept.size() > 100) kept.resize(100);         // keep_top_k
  const int n = (int)std::min<size_t>(kept.size(), 256);
  for (int i = 0; i < n; i++) {                    // objectdetect_cnn (model.cpp:362-389), facedetect_cnn's short casts (:420-434)
    const float score = kept[i].first;
    const FdBox &b = kept[i].second;
    int v[15];
    v[0] = fd_cvtt(score * score * 100);
    v[1] = fd_cvtt(b.xmin * g.W + 0.5f);
    v[2] = fd_cvtt(b.ymin * g.H + 0.5f);
    v[3] = fd_cvtt((b.xmax - b.xmin) * g.W + 0.5f);
    v[4] = fd_cvtt((b.ymax - b.ymin) * g.H + 0.5f);
    for (int lm = 0; lm < 5; lm++) {
      v[5 + lm * 2] = fd_cvtt(b.lm[lm * 2] * g.W + 0.5f);
      v[6 + lm * 2] = fd_cvtt(b.lm[lm * 2 + 1] * g.H + 0.5f);
    }
    for (int k = 0; k < 15; k++) faces[i * 15 + k] = (int16_t)v[k];
  }
  *n_faces = n;
  return B2F_OK;
}

#undef FD_MIN
#undef FD_MAX

static int fd_check(const char *who, const b2f_facedet_model *m, int n, int W, int H) {
  if (!m) { set_error("%s: NULL model", who); return B2F_EINVAL; }
  if (n <= 0 || W <= 0 || H <= 0) { set_error("%s: bad size %d x %dx%d", who, n, W, H); return B2F_EINVAL; }
  if ((long long)W * H * 3 > 2147483647LL) { set_error("%s: %dx%d overflows the int indexing of the reference", who, W, H); return B2F_EUNSUP; }
  return B2F_OK;
}

// Device scratch, tail and outputs of n frames already on the device.  layer_max [n][16], records [n][cand_cap][17] and
// n_cand [n] are optional.
static int fd_run(b2f_ctx *ctx, const b2f_facedet_model *m, const uint8_t *d_rgb, int n, int W, int H, int *n_faces, int32_t *faces,
                  int32_t *layer_max, int32_t *cand, int cand_cap, int *n_cand, cudaStream_t st) {
  FdHostOut ho;
  int rc = fd_device(ctx, m, d_rgb, n, W, H, ho, st);
  if (rc != B2F_OK) return rc;
  const FdGeom g = fd_geom(W, H);
  size_t off = 0;
  for (int f = 0; f < n; f++) {
    const int c = std::min(ho.count[f], ho.cap);
    const int32_t *r = ho.rec.data() + off * FD_REC;
    off += c;
    if (layer_max) std::copy(ho.lmax.begin() + (size_t)f * FD_NRELU, ho.lmax.begin() + (size_t)(f + 1) * FD_NRELU, layer_max + (size_t)f * FD_NRELU);
    if (n_cand) n_cand[f] = c;
    if (cand) {                                    // the records in prior order
      std::vector<int> o(c);
      for (int i = 0; i < c; i++) o[i] = i;
      std::sort(o.begin(), o.end(), [&](int a, int b) { return r[(size_t)a * FD_REC] < r[(size_t)b * FD_REC]; });
      for (int i = 0; i < std::min(c, cand_cap); i++)
        std::copy(r + (size_t)o[i] * FD_REC, r + (size_t)(o[i] + 1) * FD_REC, cand + ((size_t)f * cand_cap + i) * FD_REC);
    }
    int32_t *fo = faces + (size_t)f * 256 * 15;
    std::fill(fo, fo + 256 * 15, 0);
    n_faces[f] = 0;
    if (g.n_run == FD_NRELU && (rc = fd_tail(m, g, ho.st[f], r, c, n_faces + f, fo)) != B2F_OK) return rc;
  }
  return B2F_OK;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_facedet_model_create(b2f_ctx *ctx, const b2f_conv_layer *layers, int n_layers, b2f_facedet_model **model) {
  if (!ctx || !layers || !model) { set_error("b2f_facedet_model_create: bad argument"); return B2F_EINVAL; }
  *model = nullptr;
  if (n_layers != FD_NL) { set_error("b2f_facedet_model_create: %d layers, the network has %d", n_layers, FD_NL); return B2F_EINVAL; }
  for (int l = 0; l < FD_NL; l++) {
    const b2f_conv_layer &L = layers[l];
    const FdShape &S = FD_SHAPE[l];
    if (!L.weights || !L.bias) { set_error("b2f_facedet_model_create: layer %d has no weights or bias", l); return B2F_EINVAL; }
    if (L.kernel_size != S.k || L.channels != S.c || L.num != S.n) {
      set_error("b2f_facedet_model_create: layer %d is %dx%d, %d -> %d; the network needs %dx%d, %d -> %d", l, L.kernel_size,
                L.kernel_size, L.channels, L.num, S.k, S.k, S.c, S.n);
      return B2F_EINVAL;
    }
    // layer 0's pad and stride are not read (init_parameters runs it as a 1x1 convolution over the image blob)
    if (l > 0 && (L.stride != 1 || L.pad != (S.k == 3 ? 1 : 0))) {
      set_error("b2f_facedet_model_create: layer %d has stride %d pad %d; the network needs stride 1 pad %d", l, L.stride, L.pad, S.k == 3 ? 1 : 0);
      return B2F_EINVAL;
    }
  }
  b2f_facedet_model *m = new b2f_facedet_model();
  m->device = ctx->device;
  for (int l = 0; l < FD_NL; l++) m->fscale[l] = layers[l].scale;
  // host image of the device block
  std::vector<char> img;
  auto put = [&](const void *p, size_t bytes) { const size_t o = img.size(); img.resize(align256(o + bytes)); if (p) std::memcpy(img.data() + o, p, bytes); return o; };
  std::vector<int8_t> w0(32 * 27);
  for (int n = 0; n < 32; n++)
    for (int c = 0; c < 3; c++)
      for (int t = 0; t < 9; t++) w0[n * 27 + t * 3 + c] = layers[0].weights[(n * 3 + c) * 9 + t];
  const size_t o_w0 = put(w0.data(), w0.size()), o_b0 = put(layers[0].bias, 32 * 4);
  size_t o_w[19], o_b[19];
  for (int gi = 0; gi < 19; gi++) {
    FdGemm &G = m->g[gi];
    const int la = gi < 15 ? gi + 1 : 16 + 2 * (gi - 15), nparts = gi < 15 ? 1 : 2;
    const FdShape &S = FD_SHAPE[la];
    G.ks = S.k; G.C = S.c; G.N = 0;
    for (int p = 0; p < nparts; p++) G.N += FD_SHAPE[la + p].n;
    G.nt = G.N % 32 == 0 ? 4 : 2;
    G.Npad = (G.N + 8 * G.nt - 1) / (8 * G.nt) * (8 * G.nt);
    const int K = S.k * S.k * S.c;
    G.Kpad = (K + 31) / 32 * 32;
    std::vector<int8_t> w((size_t)G.Npad * G.Kpad, 0);
    std::vector<int32_t> b(G.Npad, 0);
    int nn = 0;
    for (int p = 0; p < nparts; p++) {
      const b2f_conv_layer &L = layers[la + p];
      for (int o = 0; o < L.num; o++, nn++) {
        b[nn] = L.bias[o];
        for (int c = 0; c < S.c; c++)
          for (int t = 0; t < S.k * S.k; t++) w[(size_t)nn * G.Kpad + t * S.c + c] = L.weights[((size_t)o * S.c + c) * S.k * S.k + t];
      }
    }
    o_w[gi] = put(w.data(), w.size());
    o_b[gi] = put(b.data(), b.size() * 4);
  }
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e == cudaSuccess) e = cudaMalloc(&m->mem, img.size());
  if (e == cudaSuccess) e = cudaMemcpy(m->mem, img.data(), img.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (m->mem) cudaFree(m->mem);
    delete m;
    set_error("b2f_facedet_model_create: %s", cudaGetErrorString(e));
    return B2F_ECUDA;
  }
  char *base = static_cast<char *>(m->mem);
  m->w0 = reinterpret_cast<int8_t *>(base + o_w0);
  m->b0 = reinterpret_cast<int32_t *>(base + o_b0);
  for (int gi = 0; gi < 19; gi++) {
    m->g[gi].w = reinterpret_cast<int8_t *>(base + o_w[gi]);
    m->g[gi].bias = reinterpret_cast<int32_t *>(base + o_b[gi]);
  }
  *model = m;
  return B2F_OK;
}

void b2f_facedet_model_free(b2f_facedet_model *model) {
  if (!model) return;
  cudaSetDevice(model->device);
  cudaFree(model->mem);
  delete model;
}

int b2f_facedet_host_r32(b2f_ctx *ctx, const b2f_facedet_model *model, const int32_t *x, size_t x_len, int width, int height,
                         int step, int *n_faces, int32_t *faces) {
  if (!ctx || !model || !n_faces || !faces || (!x && x_len)) { set_error("b2f_facedet_host_r32: bad argument"); return B2F_EINVAL; }
  if (width <= 0 || height <= 0) { *n_faces = 0; return B2F_OK; }   // the reference's first convolution fails: 0 faces
  int rc = fd_check("b2f_facedet_host_r32", model, 1, width, height);
  if (rc != B2F_OK) return rc;
  if (step != 3 * width) { set_error("b2f_facedet_host_r32: step %d, the frame needs step = 3 * width = %d", step, 3 * width); return B2F_EINVAL; }
  const size_t n = (size_t)width * height * 3;
  if (x_len < n) { set_error("b2f_facedet_host_r32: %zu values, a %dx%d RGB frame needs %zu", x_len, width, height, n); return B2F_EINVAL; }
  B2F_CUDA(cudaSetDevice(ctx->device));
  if ((rc = arena_reserve(ctx, facedet_scratch_bytes(width, height, 1) + align256(n * 4) + align256(n))) != B2F_OK) return rc;
  int32_t *d_raw = ctx->arena.get<int32_t>(n);
  uint8_t *d_rgb = ctx->arena.get<uint8_t>(n);
  B2F_ARENA_CHECK(ctx);
  cudaStream_t st = ctx->stream;
  B2F_CUDA(cudaMemcpyAsync(d_raw, x, n * 4, cudaMemcpyHostToDevice, st));
  narrow_i32_to_u8_kernel<<<(unsigned)((n + 1023) / 1024), 256, 0, st>>>(d_raw, d_rgb, n);
  B2F_LAUNCH_CHECK(ctx);
  return fd_run(ctx, model, d_rgb, 1, width, height, n_faces, faces, nullptr, nullptr, 0, nullptr, st);
}

int b2f_facedet_batch_rgb(b2f_ctx *ctx, const b2f_facedet_model *model, const uint8_t *frames, int n_frames, int width, int height,
                          int *n_faces, int32_t *faces) {
  if (!ctx || !frames || !n_faces || !faces) { set_error("b2f_facedet_batch_rgb: bad argument"); return B2F_EINVAL; }
  int rc = fd_check("b2f_facedet_batch_rgb", model, n_frames, width, height);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  const size_t fb = (size_t)width * height * 3;
  const size_t per = facedet_scratch_bytes(width, height, 1) + fb;
  const int C = (int)std::max<size_t>(1, std::min<size_t>((size_t)n_frames, FD_CHUNK_SCRATCH / per));
  if ((rc = arena_reserve(ctx, facedet_scratch_bytes(width, height, C) + 2 * align256(fb * C))) != B2F_OK) return rc;
  uint8_t *d_in[2] = {ctx->arena.get<uint8_t>(fb * C), ctx->arena.get<uint8_t>(fb * C)};
  B2F_ARENA_CHECK(ctx);
  cudaStream_t st = ctx->stream;
  const int NCH = ceil_div(n_frames, C);
  if ((rc = pipe_prepare(ctx, NCH)) != B2F_OK) return rc;
  // the upload of chunk c+1 (copy-in stream) overlaps the kernels and the host tail of chunk c
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
    if (c + 1 < NCH) {
      // chunk c+1 overwrites the buffer chunk c-1 read: that chunk's kernels finished before its tail ran
      if ((rc = upload(c + 1)) != B2F_OK) break;
    }
    rc = fd_run(ctx, model, d_in[c & 1], nf, width, height, n_faces + f0, faces + (size_t)f0 * 256 * 15, nullptr, nullptr, 0, nullptr, st);
  }
  if (rc == B2F_ECUDA && cudaPeekAtLastError() != cudaSuccess)
    set_error("b2f_facedet_batch_rgb: %s", cudaGetErrorString(cudaGetLastError()));
  const int rd = pipe_drain(ctx);
  return rc != B2F_OK ? rc : rd;
}

int b2f_facedet_dev(b2f_ctx *ctx, const b2f_facedet_model *model, const uint8_t *d_frames, int n_frames, int width, int height,
                    int *n_faces, int32_t *faces, int32_t *layer_max, int32_t *cand, int cand_cap, int *n_cand, void *stream) {
  if (!ctx || !d_frames || !n_faces || !faces || (cand && (!n_cand || cand_cap <= 0))) { set_error("b2f_facedet_dev: bad argument"); return B2F_EINVAL; }
  int rc = fd_check("b2f_facedet_dev", model, n_frames, width, height);
  if (rc != B2F_OK) return rc;
  B2F_CUDA(cudaSetDevice(ctx->device));
  cudaStream_t st;
  if ((rc = stream_handoff(ctx, stream, &st)) != B2F_OK) return rc;
  if ((rc = arena_reserve(ctx, facedet_scratch_bytes(width, height, n_frames))) != B2F_OK) return rc;
  return fd_run(ctx, model, d_frames, n_frames, width, height, n_faces, faces, layer_max, cand, cand_cap, n_cand, st);
}

}  // extern "C"
