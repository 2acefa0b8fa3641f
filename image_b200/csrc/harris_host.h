// harris_host.h — internal interface between the Harris kernels (harris.cu) and the C ABI
// (harris_api.cu).
#pragma once
#include "common.cuh"
namespace b2f {
bool harris_fused_supported(int nx, int ny, float sigma_d, float sigma_i, int gaussian);
int harris_response_device(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny,
                           const b2f_harris_params *p, int exact, float *d_R, cudaStream_t st);
// fused kernel (harris_fused.cu); d_eps: optional zero-filled per-8x8-block error bound of R; corners_only: pixels whose
// reference response is certainly below the threshold may be stored as -FLT_MAX
int harris_fused_launch(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny, const b2f_harris_params *p,
                        float *d_R, unsigned *d_eps, bool corners_only, cudaStream_t st);
int harris_taps_double(float sigma, double *B);
// certified fast path (harris.cu): reference-identical corner lists from the fused kernel + exact patches
bool harris_certified_supported(int nx, int ny, const b2f_harris_params *p);
size_t harris_certified_scratch_bytes(int n_frames, int nx, int ny, int cap, bool want_m9);
int harris_corners_certified(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny,
                             const b2f_harris_params *p, int cap, int *d_xy, float *d_strength, float *d_M9,
                             int *d_counts, float *d_R_out, cudaStream_t st);
int harris_cert_stats(b2f_ctx *ctx, unsigned long long out[4], cudaStream_t st);
// raster-ordered corner lists of frames resident on the device (output as b2f_harris_corners_dev): zero counts when no pixel
// has a full window, else the certified path where p->exact and the fused kernel allow it, else response + NMS (d_R, when
// NULL, from the arena)
int harris_corners_device(b2f_ctx *ctx, const void *d_frames, bool u8, int n_frames, int nx, int ny, const b2f_harris_params *p,
                          int cap, int *d_xy, float *d_strength, int *d_counts, float *d_R, cudaStream_t st);
int harris_nms_device(b2f_ctx *ctx, const float *d_R, int n_frames, int nx, int ny, float Th, int radius, int cap,
                      int *d_xy, float *d_strength, int *d_counts, cudaStream_t st);
// bit mask [n_frames][ny][wpr] -> exclusive per-row offsets of the set bits (row_off) and per-frame totals (d_counts)
int mask_row_offsets(b2f_ctx *ctx, const unsigned *mask, int *row_off, int *d_counts, int n_frames, int ny, int wpr, cudaStream_t st);
int harris_gather3x3(b2f_ctx *ctx, const float *d_R, const int *d_xy, float *d_M, int n, int nx, cudaStream_t st);
int harris_decimate2(b2f_ctx *ctx, const float *d_src, float *d_dst, int nx, int ny, cudaStream_t st);
int harris_double_to_float(b2f_ctx *ctx, const double *s, float *d, size_t n, cudaStream_t st);
int harris_u8_to_float(b2f_ctx *ctx, const unsigned char *s, float *d, size_t n, cudaStream_t st);
size_t harris_scratch_bytes(int n_frames, int nx, int ny, const b2f_harris_params *p, int cap);
}  // namespace b2f
