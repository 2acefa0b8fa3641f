// features.cu — Harris corners + Canny edge map + FHOG from ONE upload of each RGB frame (new surface; the three
// reference packages are separate .Call entry points that each receive their own copy of the image).
// A serving loop that wants all three pays the host->device link once: 3 B/pixel instead of 1 + 1 + 3, and the grey
// plane both Harris and Canny read is derived on the device with dlib's rule (r + g + b) / 3 (pixel.h:775-783 — the
// same grey the reference's SURF path uses, and what bench.py feeds the single-detector calls).  Frames are cut into
// chunks; the upload of chunk c+1, the kernels of chunk c and the download of chunk c-1 overlap on three streams.
// The single-detector host batches (b2f_harris_batch_u8, b2f_canny_batch, b2f_fhog_batch) run this same pipeline with
// one detector.
#include "harris_host.h"
#include <algorithm>
#include <chrono>

namespace b2f {
size_t canny_scratch_bytes(int n_frames, int nx, int ny);
int canny_device(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, int nx, int ny, double s, double low_thr,
                 double high_thr, int acc_grad, unsigned char *d_edges, int *d_nonzero, cudaStream_t st);
size_t fhog_scratch_simple(int n_frames, int rows, int cols, int cell, int frp, int fcp, int *out_nr, int *out_nc);
int fhog_device_simple(b2f_ctx *ctx, const unsigned char *d_frames, int n_frames, int rows, int cols, int cell, int frp, int fcp,
                       float *d_out, cudaStream_t st);
int fhog_check_args(const char *who, int rows, int cols, int cell, int frp, int fcp);

// 16 pixels per thread: three 16-byte loads of interleaved RGB -> one 16-byte store of grey
__global__ void __launch_bounds__(256)
rgb_to_grey_kernel(const unsigned char *__restrict__ rgb, unsigned char *__restrict__ grey, size_t n_px, int aligned) {
  const size_t i = ((size_t)blockIdx.x * 256 + threadIdx.x) * 16;
  if (i >= n_px) return;
  if (aligned && i + 16 <= n_px) {
    const uint4 a = __ldg(reinterpret_cast<const uint4 *>(rgb + 3 * i)), b = __ldg(reinterpret_cast<const uint4 *>(rgb + 3 * i) + 1),
                c = __ldg(reinterpret_cast<const uint4 *>(rgb + 3 * i) + 2);
    const unsigned w[12] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w, c.x, c.y, c.z, c.w};
    unsigned o[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {      // 4 pixels = 12 bytes = 3 words
      const unsigned w0 = w[3 * k], w1 = w[3 * k + 1], w2 = w[3 * k + 2];
      const unsigned p0 = ((w0 & 0xff) + ((w0 >> 8) & 0xff) + ((w0 >> 16) & 0xff)) / 3;
      const unsigned p1 = ((w0 >> 24) + (w1 & 0xff) + ((w1 >> 8) & 0xff)) / 3;
      const unsigned p2 = (((w1 >> 16) & 0xff) + (w1 >> 24) + (w2 & 0xff)) / 3;
      const unsigned p3 = (((w2 >> 8) & 0xff) + ((w2 >> 16) & 0xff) + (w2 >> 24)) / 3;
      o[k] = p0 | (p1 << 8) | (p2 << 16) | (p3 << 24);
    }
    *reinterpret_cast<uint4 *>(grey + i) = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    const size_t e = i + 16 < n_px ? i + 16 : n_px;
    for (size_t j = i; j < e; j++) grey[j] = (unsigned char)(((unsigned)rgb[3 * j] + rgb[3 * j + 1] + rgb[3 * j + 2]) / 3);
  }
}

int features_batch(const char *who, b2f_ctx *ctx, const uint8_t *rgb, int channels, int n_frames, int rows, int cols,
                   const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                   const b2f_canny_params *cp, uint8_t *edges, int *nonzero, int cell_size, int frp, int fcp, float *hog) {
  if (!ctx || !rgb || n_frames <= 0 || rows <= 0 || cols <= 0) { set_error("%s: bad argument", who); return B2F_EINVAL; }
  const bool do_h = hp != nullptr, do_c = cp != nullptr, do_f = cell_size > 0;
  if (do_h && (!cx || !cy || !cs || !ccounts || corner_cap <= 0)) { set_error("%s: Harris outputs missing", who); return B2F_EINVAL; }
  if (do_h && (hp->strategy != 0 || hp->precision != 0 || hp->Nscales > 1)) { set_error("%s: corners come in raster order (strategy=0, precision=0, Nscales=1)", who); return B2F_EUNSUP; }
  if (do_c && (!edges || !nonzero)) { set_error("%s: Canny outputs missing", who); return B2F_EINVAL; }
  int hnr = 0, hnc = 0, rc;
  if (do_f) {
    if ((rc = fhog_check_args(who, rows, cols, cell_size, frp, fcp)) != B2F_OK) return rc;
    if (!hog) { set_error("%s: FHOG output missing", who); return B2F_EINVAL; }
  }
  const auto t_enter = std::chrono::steady_clock::now();
  B2F_CUDA(cudaSetDevice(ctx->device));
  const int nx = cols, ny = rows;
  const size_t plane = (size_t)nx * ny, fin = plane * channels;
  // Chunk schedule: C frames per chunk, the first and the last chunk half of that — the first chunk's upload and the last
  // chunk's kernels + download are the parts nothing overlaps with (pipeline fill and drain).  Measured on 16 4K frames
  // (tools/e2e_probe.py): uniform 10.19 ms, halved ends 10.13 ms, a 1-2-4-4-2-2-1 ramp 10.92 ms.
  const int C = frames_per_chunk(ctx, fin, n_frames);
  std::vector<int> cstart;
  {
    const int edge = (C >= 2 && n_frames >= C) ? C / 2 : 0;
    std::vector<int> sizes;
    if (edge) sizes.push_back(edge);
    for (int mid = n_frames - 2 * edge; mid > 0; mid -= C) sizes.push_back(std::min(C, mid));
    if (edge) sizes.push_back(edge);
    int f = 0;
    for (int sz : sizes) { cstart.push_back(f); f += sz; }
    cstart.push_back(n_frames);
  }
  const int NCH = (int)cstart.size() - 1;
  const size_t f_scr = do_f ? fhog_scratch_simple(C, rows, cols, cell_size, frp, fcp, &hnr, &hnc) : 0;
  const size_t fout = (size_t)hnr * hnc * 31;
  // Harris scratch only where some pixel has a full window (harris_corners_device zeroes the counts of other frames)
  const int radius = do_h ? (int)(2 * hp->sigma_i + 0.5) : 0;
  const bool h_runs = do_h && !(nx < 3 || ny < 3 || ny <= 2 * radius + 1 || nx <= 2 * radius + 1);
  const bool derive_grey = channels == 3 && (do_h || do_c);
  // the detectors run side by side on three streams: each has its own scratch region
  const size_t scr_h = h_runs ? align256(harris_scratch_bytes(C, nx, ny, hp, corner_cap)) : 0;
  const size_t scr_c = do_c ? align256(canny_scratch_bytes(C, nx, ny)) : 0;
  const size_t scr = scr_h + scr_c + align256(f_scr);
  const size_t rec = (size_t)n_frames * corner_cap;
  rc = arena_reserve(ctx, scr + align256(fin * n_frames) + (derive_grey ? 2 * align256(plane * C) : 0) + (do_c ? align256(plane * n_frames) : 0) +
                              align256(fout * n_frames * 4) + 2 * align256(rec * 4) + 2 * align256((size_t)n_frames * 4) + 8192);
  if (rc != B2F_OK) return rc;
  unsigned char *d_rgb = ctx->arena.get<unsigned char>(fin * n_frames);
  unsigned char *d_grey2[2] = {nullptr, nullptr};   // derived grey planes of one chunk, double-buffered (Canny of chunk c reads while chunk c+1 is derived)
  if (derive_grey) { d_grey2[0] = ctx->arena.get<unsigned char>(plane * C); d_grey2[1] = ctx->arena.get<unsigned char>(plane * C); }
  unsigned char *d_edges = do_c ? ctx->arena.get<unsigned char>(plane * n_frames) : nullptr;
  float *d_hog = do_f && fout ? ctx->arena.get<float>(fout * n_frames) : nullptr;
  int *d_xy = do_h ? ctx->arena.get<int>(rec) : nullptr;
  float *d_s = do_h ? ctx->arena.get<float>(rec) : nullptr;
  int *d_cnt = ctx->arena.get<int>(n_frames), *d_nz = ctx->arena.get<int>(n_frames);
  B2F_ARENA_CHECK(ctx);
  const size_t mark_h = ctx->arena.off, mark_c = mark_h + scr_h, mark_f = mark_c + scr_c, mark_end = mark_f + align256(f_scr);
  cudaStream_t st = ctx->stream;
  for (cudaStream_t &s : ctx->s_aux)
    if (!s) B2F_CUDA(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking));
  cudaStream_t s_canny = ctx->s_aux[0], s_fhog = ctx->s_aux[1];
  // The head of every corner list (SPEC entries) and the counters ride home with their chunk, into pinned memory, so the
  // usual case (a few thousand corners per frame) needs no second round trip after the pipeline has drained.
  const int SPEC = std::min(corner_cap, 4096);
  int *p_xy = nullptr, *p_cnt = nullptr, *p_nz = nullptr;
  float *p_s = nullptr;
  {
    const size_t nspec = (size_t)n_frames * SPEC;
    if ((rc = pinned_reserve(ctx, nspec * 8 + (size_t)n_frames * 8)) != B2F_OK) return rc;
    p_xy = (int *)ctx->pinned;
    p_s = (float *)(p_xy + nspec);
    p_cnt = (int *)(p_s + nspec);
    p_nz = p_cnt + n_frames;
    for (int f = 0; f < n_frames; f++) p_cnt[f] = 0;
  }
  if ((rc = pipe_prepare(ctx, 5 * NCH)) != B2F_OK) return rc;
  const bool trace = getenv("B2F_FEAT_TRACE") != nullptr;
  std::vector<cudaEvent_t> tev;
  auto host_ms = [&]() { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t_enter).count(); };
  double h_first = 0, h_queued = 0;
  if (trace) {   // B2F_FEAT_TRACE=1: the timeline of this call on stderr (tools/e2e_trace.py)
    tev.resize(1 + 4 * NCH);
    for (auto &e : tev) cudaEventCreate(&e);
    cudaEventRecord(tev[0], ctx->s_in);
    h_first = host_ms();
  }
  for (int c = 0; c < NCH; c++) {
    const int f0 = cstart[c], nf = cstart[c + 1] - f0;
    cudaEvent_t e_in = ctx->events[5 * c], e_hog = ctx->events[5 * c + 1], e_canny = ctx->events[5 * c + 2], e_done = ctx->events[5 * c + 3], e_grey = ctx->events[5 * c + 4];
    unsigned char *d_grey = d_grey2[c & 1];
    rc = B2F_OK;
    if (cudaMemcpyAsync(d_rgb + fin * f0, rgb + fin * f0, fin * nf, cudaMemcpyHostToDevice, ctx->s_in) != cudaSuccess ||
        cudaEventRecord(e_in, ctx->s_in) != cudaSuccess || cudaStreamWaitEvent(st, e_in, 0) != cudaSuccess) rc = B2F_ECUDA;
    if (trace) { cudaEventRecord(tev[1 + 4 * c], ctx->s_in); cudaEventRecord(tev[2 + 4 * c], st); }
    const unsigned char *d_grey_c = channels == 1 ? d_rgb + fin * f0 : d_grey;     // grey input is used where it landed
    // Three detectors side by side: FHOG (needs only the RGB frames) on its own stream, the grey derivation and Harris on
    // the context stream, Canny on a third.  Each result starts its way home as soon as its detector has finished.
    if (rc == B2F_OK && d_hog) {
      ctx->arena.region(mark_f, mark_end);
      if (cudaStreamWaitEvent(s_fhog, e_in, 0) != cudaSuccess) rc = B2F_ECUDA;
      if (rc == B2F_OK) rc = fhog_device_simple(ctx, d_rgb + fin * f0, nf, rows, cols, cell_size, frp, fcp, d_hog + fout * f0, s_fhog);
      if (rc == B2F_OK && (cudaEventRecord(e_hog, s_fhog) != cudaSuccess || cudaStreamWaitEvent(ctx->s_out, e_hog, 0) != cudaSuccess ||
                           cudaMemcpyAsync(hog + fout * f0, d_hog + fout * f0, fout * nf * 4, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess)) rc = B2F_ECUDA;
    }
    if (rc == B2F_OK && derive_grey) {
      const size_t npx = plane * nf;
      const int al = ((reinterpret_cast<uintptr_t>(d_rgb + fin * f0) | reinterpret_cast<uintptr_t>(d_grey)) & 15) == 0;
      if (do_c && c >= 2 && cudaStreamWaitEvent(st, ctx->events[5 * (c - 2) + 2], 0) != cudaSuccess) rc = B2F_ECUDA;   // Canny of chunk c-2 read this buffer
      rgb_to_grey_kernel<<<(unsigned)((npx + 4095) / 4096), 256, 0, st>>>(d_rgb + fin * f0, d_grey, npx, al);
      ctx->launches++;
      if (cudaGetLastError() != cudaSuccess) rc = B2F_ECUDA;
    }
    if (rc == B2F_OK && do_c) {
      ctx->arena.region(mark_c, mark_f);
      if (cudaEventRecord(e_grey, st) != cudaSuccess || cudaStreamWaitEvent(s_canny, e_grey, 0) != cudaSuccess) rc = B2F_ECUDA;
      if (rc == B2F_OK) rc = canny_device(ctx, d_grey_c, nf, nx, ny, cp->s, cp->low_thr, cp->high_thr, cp->acc_grad, d_edges + plane * f0, d_nz + f0, s_canny);
      if (rc == B2F_OK && (cudaEventRecord(e_canny, s_canny) != cudaSuccess || cudaStreamWaitEvent(ctx->s_out, e_canny, 0) != cudaSuccess ||
                           cudaMemcpyAsync(edges + plane * f0, d_edges + plane * f0, plane * nf, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess ||
                           cudaMemcpyAsync(p_nz + f0, d_nz + f0, sizeof(int) * nf, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess)) rc = B2F_ECUDA;
    }
    if (rc == B2F_OK && do_h) {
      ctx->arena.region(mark_h, mark_c);
      rc = harris_corners_device(ctx, d_grey_c, true, nf, nx, ny, hp, corner_cap, d_xy + (size_t)f0 * corner_cap, d_s + (size_t)f0 * corner_cap,
                                 d_cnt + f0, nullptr, st);
    }
    if (rc == B2F_OK && (cudaEventRecord(e_done, st) != cudaSuccess || cudaStreamWaitEvent(ctx->s_out, e_done, 0) != cudaSuccess)) rc = B2F_ECUDA;
    if (trace) cudaEventRecord(tev[3 + 4 * c], st);
    if (rc == B2F_OK && do_h && SPEC > 0 &&
        (cudaMemcpy2DAsync(p_xy + (size_t)f0 * SPEC, (size_t)SPEC * 4, d_xy + (size_t)f0 * corner_cap, (size_t)corner_cap * 4, (size_t)SPEC * 4, nf, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess ||
         cudaMemcpy2DAsync(p_s + (size_t)f0 * SPEC, (size_t)SPEC * 4, d_s + (size_t)f0 * corner_cap, (size_t)corner_cap * 4, (size_t)SPEC * 4, nf, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess)) rc = B2F_ECUDA;
    if (rc == B2F_OK && do_h && cudaMemcpyAsync(p_cnt + f0, d_cnt + f0, sizeof(int) * nf, cudaMemcpyDeviceToHost, ctx->s_out) != cudaSuccess) rc = B2F_ECUDA;
    if (trace) cudaEventRecord(tev[4 + 4 * c], ctx->s_out);
    if (rc != B2F_OK) {
      if (rc == B2F_ECUDA) set_error("%s: CUDA error in chunk %d: %s", who, c, cudaGetErrorString(cudaGetLastError()));
      pipe_drain(ctx);
      return rc;
    }
  }
  if (trace) h_queued = host_ms();
  if ((rc = pipe_drain(ctx)) != B2F_OK) return rc;
  if (trace) {
    fprintf(stderr, "host: first upload queued at %.3f ms after entry, all chunks queued at %.3f, drained at %.3f\n", h_first, h_queued, host_ms());
    for (int c = 0; c < NCH; c++) {
      float t[4];
      for (int k = 0; k < 4; k++) cudaEventElapsedTime(&t[k], tev[0], tev[1 + 4 * c + k]);
      fprintf(stderr, "chunk %2d (%d frames): upload done %.3f  compute %.3f .. %.3f  download done %.3f ms\n", c, cstart[c + 1] - cstart[c], t[0], t[1], t[2], t[3]);
    }
    for (auto &e : tev) cudaEventDestroy(e);
  }
  if (do_c) for (int f = 0; f < n_frames; f++) nonzero[f] = p_nz[f];
  if (!do_h) return B2F_OK;
  // A count of -1: the certified path had more candidates than corner_cap record slots (it sizes them by the caller's cap),
  // so its list and count are unknown — although the frame may have no more than corner_cap corners — or a corner ties
  // its left neighbour exactly, which only the reference's row scan settles.  Such frames run again through the staged
  // kernels, whose NMS counts every corner; the grey plane of an RGB frame is derived once more from d_rgb, which still
  // holds the whole batch.
  for (int f = 0; f < n_frames; f++) {
    if (p_cnt[f] >= 0) continue;
    ctx->arena.region(mark_h, mark_c);
    const unsigned char *g = d_rgb + fin * f;
    if (channels == 3) {
      const int al = ((reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(d_grey2[0])) & 15) == 0;
      rgb_to_grey_kernel<<<(unsigned)((plane + 4095) / 4096), 256, 0, st>>>(g, d_grey2[0], plane, al);
      B2F_LAUNCH_CHECK(ctx);
      g = d_grey2[0];
    }
    b2f_harris_params q = *hp;
    q.exact = 1;
    const size_t o = (size_t)f * corner_cap;
    if ((rc = harris_corners_device(ctx, g, true, 1, nx, ny, &q, corner_cap, d_xy + o, d_s + o, d_cnt + f, nullptr, st)) != B2F_OK) return rc;
    if (SPEC > 0) {
      B2F_CUDA(cudaMemcpyAsync(p_xy + (size_t)f * SPEC, d_xy + o, sizeof(int) * SPEC, cudaMemcpyDeviceToHost, st));
      B2F_CUDA(cudaMemcpyAsync(p_s + (size_t)f * SPEC, d_s + o, sizeof(float) * SPEC, cudaMemcpyDeviceToHost, st));
    }
    B2F_CUDA(cudaMemcpyAsync(p_cnt + f, d_cnt + f, sizeof(int), cudaMemcpyDeviceToHost, st));
    B2F_CUDA(cudaStreamSynchronize(st));
  }
  bool over = false, deep = false;
  for (int f = 0; f < n_frames; f++) {
    int m = p_cnt[f];
    if (m < 0) { over = true; m = corner_cap + 1; }
    ccounts[f] = m;
    over |= m > corner_cap;
    m = std::min(m, corner_cap);
    deep |= m > SPEC;
    const size_t o = (size_t)f * corner_cap, po = (size_t)f * SPEC;
    for (int i = 0; i < std::min(m, SPEC); i++) { const int q = p_xy[po + i]; cx[o + i] = (float)(q % nx); cy[o + i] = (float)(q / nx); cs[o + i] = p_s[po + i]; }
  }
  if (deep) {   // frames with more than SPEC corners: fetch the rest of their lists (the pinned block is free again by now)
    if ((rc = pinned_reserve(ctx, rec * 8)) != B2F_OK) return rc;
    int *h_xy = (int *)ctx->pinned;
    float *h_s = (float *)(h_xy + rec);
    for (int f = 0; f < n_frames; f++) {
      const int m = std::min(ccounts[f], corner_cap);
      if (m <= SPEC) continue;
      const size_t o = (size_t)f * corner_cap + SPEC;
      B2F_CUDA(cudaMemcpyAsync(h_xy + o, d_xy + o, sizeof(int) * (m - SPEC), cudaMemcpyDeviceToHost, st));
      B2F_CUDA(cudaMemcpyAsync(h_s + o, d_s + o, sizeof(float) * (m - SPEC), cudaMemcpyDeviceToHost, st));
    }
    B2F_CUDA(cudaStreamSynchronize(st));
    for (int f = 0; f < n_frames; f++) {
      const int m = std::min(ccounts[f], corner_cap);
      const size_t o = (size_t)f * corner_cap;
      for (int i = SPEC; i < m; i++) { const int q = h_xy[o + i]; cx[o + i] = (float)(q % nx); cy[o + i] = (float)(q / nx); cs[o + i] = h_s[o + i]; }
    }
  }
  if (over) { set_error("%s: at least one frame has more than corner_cap=%d corners", who, corner_cap); return B2F_ECAP; }
  return B2F_OK;
}

}  // namespace b2f

using namespace b2f;

extern "C" {

int b2f_features_batch_rgb(b2f_ctx *ctx, const uint8_t *rgb, int n_frames, int rows, int cols,
                           const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                           const b2f_canny_params *cp, uint8_t *edges, int *nonzero,
                           int cell_size, int frp, int fcp, float *hog) {
  return features_batch("b2f_features_batch_rgb", ctx, rgb, 3, n_frames, rows, cols, hp, corner_cap, cx, cy, cs, ccounts, cp, edges, nonzero,
                        cell_size, frp, fcp, hog);
}

// grey u8 frames [n][ny][nx]: Harris corners + Canny edge map from one upload (BASELINE.json config 5's stream)
int b2f_features_batch_grey(b2f_ctx *ctx, const uint8_t *grey, int n_frames, int nx, int ny,
                            const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                            const b2f_canny_params *cp, uint8_t *edges, int *nonzero) {
  return features_batch("b2f_features_batch_grey", ctx, grey, 1, n_frames, ny, nx, hp, corner_cap, cx, cy, cs, ccounts, cp, edges, nonzero,
                        0, 0, 0, nullptr);
}

}  // extern "C"
