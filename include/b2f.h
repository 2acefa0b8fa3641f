/* b2f.h — C ABI of libb200feat.so, the H100-native (sm_90a) replacement for the per-pixel
 * hot path of bnosac/image's image.CornerDetectionHarris, image.CannyEdges and image.dlib
 * (FHOG / SURF).  Plain C: pointers and sizes only, no C++ / torch / R types.
 *
 * Each `*_host` entry point is what the body of one reference Rcpp export reduces to
 * (INTEGRATION.md shows the four replacement bodies):
 *   b2f_harris_host  <- detect_corners        image.CornerDetectionHarris/src/rcpp_harris.cpp:19-59
 *   b2f_canny_host   <- canny_edge_detector   image.CannyEdges/src/rcpp_canny.cpp:122-245
 *   b2f_fhog_host    <- dlib_fhog             image.dlib/src/rcpp_fhog.cpp:10-46
 *   b2f_surf_host    <- dlib_surf_points      image.dlib/src/rcpp_surf.cpp:10-54
 * The `*_batch` forms take n_frames equally-sized frames in HOST memory (new surface: the
 * reference has no batch API; a single call is batch = 1) and the `*_dev` forms take frames
 * already resident in HBM plus a CUDA stream (benchmark / pipeline use).
 *
 * Conventions
 *   - images are row-major with x fastest: pixel (x,y) at [y*nx + x]  (nx = R's nrow)
 *   - every function returns B2F_OK (0) or a negative B2F_E* code; b2f_last_error() gives the
 *     thread-local message.  Nothing longjmps or throws across this boundary.
 *   - buffers returned through `float **` / `double **` are malloc'ed by the library and are
 *     released with b2f_free(); no pointer is retained after a call returns.
 *   - the library never falls back to a CPU path: if no CUDA device is usable b2f_init fails.
 */
#ifndef B2F_H
#define B2F_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2F_OK 0
#define B2F_EINVAL (-1)   /* bad argument */
#define B2F_ECUDA (-2)    /* CUDA runtime error (message has the cudaError string) */
#define B2F_ENOMEM (-3)
#define B2F_ECAP (-4)     /* caller-provided capacity too small (counts still reported) */
#define B2F_EUNSUP (-5)   /* parameter combination not supported on the GPU path */

typedef struct b2f_ctx b2f_ctx;   /* one per (host thread, device): stream + scratch arena */

/* lifecycle — called from R_init_<pkg> / .onUnload in the R packages (INTEGRATION.md) */
int b2f_init(int device, b2f_ctx **ctx);
void b2f_shutdown(b2f_ctx *ctx);
const char *b2f_last_error(void);
const char *b2f_version(void);
int b2f_device_count(void);
void b2f_free(void *p);
/* the CUDA stream (cudaStream_t) this context launches on, for callers that time with events */
void *b2f_stream(b2f_ctx *ctx);
/* kernels launched by this context since creation (bench.py reports it as gpu_launches) */
long long b2f_launch_count(b2f_ctx *ctx);
/* The host batch calls (*_batch) cut their frames into chunks of about `bytes` input bytes (default 48 MiB)
 * so that the upload of chunk c+1, the kernels of chunk c and the download of chunk c-1 overlap. */
int b2f_set_chunk_bytes(b2f_ctx *ctx, size_t bytes);

/* ------------------------------------------------------------------------------ Harris ----
 * Integer fields carry the C++ meaning seen at the .Call boundary (gaussian.h:14-16,
 * gradient.h:14-15, harris.h:16-24, interpolation.h:13-15):
 *   gaussian 0=STD 1=SII("fast") 2=none; gradient 0=central 1=Sobel; measure 0=Harris
 *   1=Shi-Tomasi 2=harmonic mean; strategy 0=all 1=sorted 2=N best 3=N distributed;
 *   precision 0=none 1=quadratic 2=quartic.                                                  */
typedef struct {
  float k, sigma_d, sigma_i, threshold;
  int gaussian, gradient, strategy, Nselect, measure, Nscales, precision, cells, verbose;
  /* not a reference argument.
   * 0 (default) = certified fast path: the fused fp32 kernel proposes key points together with a bound on its
   *     distance from the reference's R; every proposed key point is re-evaluated with the reference's own
   *     arithmetic on a small patch, so the lists (positions, order) and strengths are the reference's bit for
   *     bit.  Parameter sets the fused kernel does not cover run the staged kernels instead (same results).
   * 1 = staged kernels that repeat the reference's double-accumulate arithmetic over whole planes.
   * 2 = fused fp32 kernel + plain NMS, uncertified: R within 1e-4, lists identical except at float near-ties. */
  int exact;
} b2f_harris_params;
void b2f_harris_default_params(b2f_harris_params *p);   /* defaults of rcpp_harris.cpp:19-32 */

/* detect_corners: img = nx*ny floats (the reference narrows R's doubles to float first,
 * rcpp_harris.cpp:35).  Outputs three malloc'ed arrays of *n floats (x, y, strength). */
int b2f_harris_host(b2f_ctx *ctx, const float *img, int nx, int ny, const b2f_harris_params *p,
                    float **x, float **y, float **strength, int *n);

/* batch of u8 frames in host memory; per frame at most `cap` corners are written at
 * x[f*cap + i] ...; counts[f] is the true count (B2F_ECAP if any exceeds cap). */
int b2f_harris_batch_u8(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int nx, int ny,
                        const b2f_harris_params *p, int cap, float *x, float *y, float *strength,
                        int *counts);

/* device-resident stages.  d_frames: n_frames planes of nx*ny u8 (is_u8=1) or float (0) in HBM.
 * d_R: n_frames*nx*ny floats.  Asynchronous on `stream` (cudaStream_t; NULL = ctx stream). */
int b2f_harris_response_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                            const b2f_harris_params *p, float *d_R, void *stream);
/* Frames resident in HBM -> reference-identical corner lists, all on the device and asynchronous on `stream`:
 * d_xy[f*cap + i] = y*nx + x (raster order, harris.cpp:250-252), d_strength the reference's R there,
 * d_counts[f] the number of corners (may exceed cap: only cap are stored; -1 = the certified path could not settle the
 * frame's list: its candidate records, sized by cap, overflowed, or a corner ties its left neighbour exactly, where the
 * reference's row scan decides; rerun with a larger cap or with params.exact = 1).  d_R (optional, n_frames*nx*ny floats) receives the fp32 response planes of the
 * certified path, in which pixels whose reference response is certainly below the threshold may hold -FLT_MAX
 * (b2f_harris_response_dev / _eps_dev return the plain planes).
 * strategy / precision / Nscales of `p` are not applied here (b2f_harris_host does them per frame). */
int b2f_harris_corners_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                           const b2f_harris_params *p, int cap, int *d_xy, float *d_strength, int *d_counts,
                           float *d_R, void *stream);
/* certification counters of this context since b2f_init: out4 = {candidates proposed by the tolerant NMS,
 * of which undecided (full window recomputed exactly), violations of the error bound (must be 0), kept}. */
int b2f_harris_cert_stats(b2f_ctx *ctx, unsigned long long *out4);
/* diagnostics: fused response plus its per-8x8-block error bound (d_eps: n_frames*ceil(ny/8)*ceil(nx/8) floats) */
int b2f_harris_response_eps_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int nx, int ny,
                                const b2f_harris_params *p, float *d_R, float *d_eps, void *stream);
/* NMS + raster-ordered compaction on device: d_xy receives y*nx+x (int32), d_strength the R
 * value, d_counts[f] the number of corners of frame f (may exceed cap; only cap are stored). */
int b2f_harris_nms_dev(b2f_ctx *ctx, const float *d_R, int n_frames, int nx, int ny, float threshold,
                       int radius, int cap, int *d_xy, float *d_strength, int *d_counts, void *stream);

/* ------------------------------------------------------------------------------- Canny ----
 * canny_edge_detector: img = nx*ny u8 (R's ints are narrowed to unsigned char,
 * rcpp_canny.cpp:137); low/high thresholds are truncated to int exactly like the reference
 * (rcpp_canny.cpp:88,180).  edges = nx*ny bytes, 0 or 255; *nonzero = number of 255s. */
int b2f_canny_host(b2f_ctx *ctx, const uint8_t *img, int nx, int ny, double s, double low_thr,
                   double high_thr, int acc_grad, uint8_t *edges, int *nonzero);
int b2f_canny_batch(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int nx, int ny, double s,
                    double low_thr, double high_thr, int acc_grad, uint8_t *edges, int *nonzero);
int b2f_canny_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int nx, int ny, double s,
                  double low_thr, double high_thr, int acc_grad, uint8_t *d_edges, int *d_nonzero,
                  void *stream);
/* Canny hysteresis on given class maps (the stage after NMS): d_cls = n_frames*ny*nx bytes; a pixel is an edge
 * candidate iff its byte is non-zero and strong iff it is 2 (rcpp_canny.cpp:184-215).  Output as b2f_canny_dev.
 * Runs the same hysteresis kernels as b2f_canny_dev (stage-level testing). */
int b2f_canny_hysteresis_dev(b2f_ctx *ctx, const uint8_t *d_cls, int n_frames, int nx, int ny,
                             uint8_t *d_edges, int *d_nonzero, void *stream);

/* pixels of this context's Canny calls that the fp32 tier could not certify and the exact fp64 tier decided (since b2f_init) */
int b2f_canny_stats(b2f_ctx *ctx, unsigned long long *tier2_pixels);

/* -------------------------------------------------------------------------------- FHOG ----
 * dlib_fhog: rgb = rows*cols*3 interleaved u8 (x[3*c + 3*cols*r + ch], rcpp_fhog.cpp:19-23).
 * Output `hog` is [hog_nr][hog_nc][31] floats (row, col, feature) — the element order of
 * dlib's array2d<matrix<float,31,1>>; the Rcpp shim transposes to R's y + nr*(x + nc*feat).
 * b2f_fhog_size gives the output shape for given inputs (fhog.h:790-813, init_hog :448-471).
 * Every cell_size >= 1 is served: cell_size == 1 takes dlib's separate routine (fhog.h:495-694), like the
 * reference's extract_fhog_features does (fhog.h:1099-1113). */
int b2f_fhog_size(int rows, int cols, int cell_size, int filter_rows_padding, int filter_cols_padding,
                  int *hog_nr, int *hog_nc);
int b2f_fhog_host(b2f_ctx *ctx, const uint8_t *rgb, int rows, int cols, int cell_size,
                  int filter_rows_padding, int filter_cols_padding, float *hog);
int b2f_fhog_batch(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int rows, int cols, int cell_size,
                   int filter_rows_padding, int filter_cols_padding, float *hog);
int b2f_fhog_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int rows, int cols, int cell_size,
                 int filter_rows_padding, int filter_cols_padding, float *d_hog, void *stream);

/* -------------------------------------------------------------------------------- SURF ----
 * dlib_surf_points: same input layout as FHOG.  One record per key point, in the order the
 * reference returns them (score descending, surf.h:268-285). */
typedef struct {
  double x, y;          /* interest_point::center */
  double angle;         /* surf_point::angle */
  double scale;         /* interest_point::scale   (R: pyramid_scale) */
  double score;         /* interest_point::score */
  double laplacian;     /* +1 / -1 */
  double des[64];       /* surf_point::des */
} b2f_surf_point;
int b2f_surf_host(b2f_ctx *ctx, const uint8_t *rgb, int rows, int cols, long max_points,
                  double detection_threshold, b2f_surf_point **points, int *n);
int b2f_surf_batch(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int rows, int cols, long max_points,
                   double detection_threshold, int cap, b2f_surf_point *points, int *counts);
/* frames resident in HBM (new surface); the records land in host memory like b2f_surf_batch's (the sort / filter tail
 * of get_surf_points, surf.h:268-285, runs on the host).  Synchronous. */
int b2f_surf_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int rows, int cols, long max_points,
                 double detection_threshold, int cap, b2f_surf_point *points, int *counts, void *stream);

/* ---------------------------------------------------------------- R payloads as they are ----
 * SURVEY.md 8f rank 4: the vectors the reference's Rcpp exports receive (R `double` for detect_corners, rcpp_harris.cpp:19-35;
 * R `integer` for canny_edge_detector :122-137, dlib_fhog rcpp_fhog.cpp:10-24, dlib_surf_points rcpp_surf.cpp:10-24) are
 * uploaded untouched and narrowed ON THE DEVICE with the reference's conversions ((float)double, (unsigned char)int)
 * instead of in scalar host loops.  Same results as the *_host forms on the narrowed data. */
int b2f_harris_host_r64(b2f_ctx *ctx, const double *img, int nx, int ny, const b2f_harris_params *p,
                        float **x, float **y, float **strength, int *n);
int b2f_canny_host_r32(b2f_ctx *ctx, const int32_t *image, int nx, int ny, double s, double low_thr, double high_thr,
                       int acc_grad, uint8_t *edges, int *nonzero);
int b2f_fhog_host_r32(b2f_ctx *ctx, const int32_t *x, int rows, int cols, int cell_size, int filter_rows_padding,
                      int filter_cols_padding, float *hog);
int b2f_surf_host_r32(b2f_ctx *ctx, const int32_t *x, int rows, int cols, long max_points, double detection_threshold,
                      b2f_surf_point **points, int *n);

/* ------------------------------------------------------------------ combined batch ----
 * New surface: Harris corners + Canny edge map + FHOG from ONE upload of each interleaved RGB frame (rows x cols x 3).
 * The grey plane Harris and Canny work on is derived on the device with dlib's rule (r + g + b) / 3 (pixel.h:775-783).
 * Results are those of the single-detector batch calls on the same frames / that grey plane.  Pass hp = NULL,
 * cp = NULL or cell_size = 0 to skip a detector.  Harris: raster-ordered corners (strategy 0, precision 0, one scale),
 * at most corner_cap per frame at [f*corner_cap + i]; Canny: edges rows*cols bytes per frame; FHOG: b2f_fhog_size floats. */
typedef struct { double s, low_thr, high_thr; int acc_grad; } b2f_canny_params;
int b2f_features_batch_rgb(b2f_ctx *ctx, const uint8_t *rgb, int n_frames, int rows, int cols,
                           const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                           const b2f_canny_params *cp, uint8_t *edges, int *nonzero,
                           int cell_size, int filter_rows_padding, int filter_cols_padding, float *hog);
/* the same for grey u8 frames [n][ny][nx]: Harris + Canny from one upload (BASELINE.json config 5's stream) */
int b2f_features_batch_grey(b2f_ctx *ctx, const uint8_t *grey, int n_frames, int nx, int ny,
                            const b2f_harris_params *hp, int corner_cap, float *cx, float *cy, float *cs, int *ccounts,
                            const b2f_canny_params *cp, uint8_t *edges, int *nonzero);

/* ------------------------------------------------------------------- ContourDetector ----
 * SURVEY.md 8f "next", rank 1: the data-parallel front end of smooth_contours() (image.ContourDetector/src/
 * smooth_contours.c: gaussian_filter :184-262, compute_gradient :339-356, compute_edge_points :427-505).
 * The reference materialises seven double planes for its sequential chainer; here the planes stay on the device
 * and the COMPACT list of edge points comes back, in raster order: idx = x + y*X, (ex, ey) the sub-pixel position
 * (Ex, Ey of the reference), (gx, gy) the gradient there (all that chain() :289-336 reads).  Every value is
 * bit-identical to the reference's doubles.  sigma <= 0 selects the reference's own sigma (:1466-1479).
 * `gauss` (optional) receives the blurred image for `diff = image - gauss` (:1498).  image[x + y*X] as in the reference.
 * b2f_contour_edge_points_host mallocs its five outputs (b2f_free); the batch / dev forms (new surface, u8 or double
 * frames) write at most `cap` records per frame at [f*cap + i] and the true count to counts[f] (B2F_ECAP if any exceeds). */
int b2f_contour_edge_points_host(b2f_ctx *ctx, const double *image, int X, int Y, double sigma, double *gauss, int **idx,
                                 double **ex, double **ey, double **gx, double **gy, int *n);
int b2f_contour_edge_points_batch_u8(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int X, int Y, double sigma, int cap,
                                     int *idx, double *ex, double *ey, double *gx, double *gy, int *counts);
int b2f_contour_edge_points_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int X, int Y, double sigma, int cap,
                                int *d_idx, double *d_ex, double *d_ey, double *d_gx, double *d_gy, int *d_counts, double *d_gauss,
                                void *stream);

/* --------------------------------------------------------------- LineSegmentDetector ----
 * SURVEY.md 8f "next", rank 2: the data-parallel front end of LineSegmentDetection() (image.LineSegmentDetector/src/
 * lsd.c: gaussian_sampler :603-720 and ll_angle :744-880, called at :2455-2462).  For an X x Y image (image[x + y*X])
 * the outputs live on the scaled grid N x M = ceil(X*scale) x ceil(Y*scale) (b2f_lsd_front_size):
 *   angles  [y*N + x]  level-line angle, or NOTDEF = -1024.0 where modgrad <= quant / sin(pi*ang_th/180)
 *   modgrad [y*N + x]  gradient modulus (0 in the last row / column, which the reference leaves unset)
 *   list               the (N-1)(M-1) gradient pixels as x + y*N, in the order of the reference's bucket list
 *                      (n_bins buckets of modgrad*n_bins/max_grad, highest first; inside a bucket x outer, y inner)
 *   scaled  (optional) the sub-sampled image.
 * modgrad, the NOTDEF pattern and the list order are bit-identical to the reference; defined angles differ from libm's
 * atan2 by at most a few ulp.  The Rcpp defaults are scale 0.8, sigma_scale 0.6, quant 2, ang_th 22.5, n_bins 1024
 * (line_segment_detector.cpp:8-21).  The `_dev` form takes n_frames u8 or double frames resident in HBM. */
int b2f_lsd_front_size(int X, int Y, double scale, int *N, int *M);
int b2f_lsd_front_host(b2f_ctx *ctx, const double *image, int X, int Y, double scale, double sigma_scale, double quant,
                       double ang_th, int n_bins, double *angles, double *modgrad, int *list, int *list_len, double *scaled);
int b2f_lsd_front_dev(b2f_ctx *ctx, const void *d_frames, int is_u8, int n_frames, int X, int Y, double scale,
                      double sigma_scale, double quant, double ang_th, int n_bins, double *d_angles, double *d_modgrad,
                      int *d_list, double *d_scaled, void *stream);

/* -------------------------------------------------------------------------------- Otsu ----
 * SURVEY.md 8f "next", rank 4.  Replaces the body of otsu() (image.Otsu/src/rcpp_otsu.cpp:166-186:
 * computeHistogram :63-81, computeOtsusSegmentation :113-163, segmentImage :88-105).
 * override_threshold 0 = compute the Otsu threshold (the reference's convention), 1..255 = use it.
 * b2f_otsu_host: `img` = the NumericVector narrowed to float (rcpp_otsu.cpp:170-172), any linear order;
 *   out = 255.0f / 0.0f per pixel, *threshold = the threshold used.  Pixel values whose (int) truncation is
 *   outside 0..255 are undefined behaviour in the reference and give B2F_EINVAL here.
 * b2f_otsu_batch_u8 / b2f_otsu_dev: new surface, u8 frames [n][height][width] in host / device memory,
 *   u8 0/255 output, one threshold per frame. */
int b2f_otsu_host(b2f_ctx *ctx, const float *img, int width, int height, int override_threshold, float *out, int *threshold);
int b2f_otsu_batch_u8(b2f_ctx *ctx, const uint8_t *frames, int n_frames, int width, int height, int override_threshold,
                      uint8_t *out, int *thresholds);
int b2f_otsu_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int width, int height, int override_threshold,
                 uint8_t *d_out, int *d_thresholds, void *stream);

/* ---------------------------------------------------------------------------- NL-means ----
 * Non-local means of image.DenoiseNLMeans (rcpp_nlmeans, image.DenoiseNLMeans/src/rcpp_denoisenlmeans.cpp, which calls
 * nlmeans_ipol in libdenoising.cpp).  Images are channel-planar: value x + width*y + width*height*c.  Output values are
 * the reference's float results bit for bit, in the order the reference computes them when run on one thread (DESIGN.md
 * §5: its OpenMP loop races on the output).  channels is mapped like the glue: 2 -> 1, above 3 -> 3; 0 or below is an error.
 * b2f_nlmeans_resolve: the glue's parameter table.  With args_auto != 0, (*win, *bloc, *filter) are set from the row of
 *   `channels` (1 = grey, else colour) and sigma; sigma <= 0 takes the last row, sigma > 100 (or NaN) returns B2F_EINVAL
 *   with the reference's message.  With args_auto == 0 the values are left as given.  Host code only, no context.
 * b2f_nlmeans_host_r32: the body of rcpp_nlmeans.  image = width*height*channels R integers, narrowed to float on the
 *   device; three equal planes are denoised as one (*out_channels = 1).  out receives *out_channels planes of floats
 *   (room for width*height*min(mapped channels) is needed); *_used are the parameters the call ran with.
 * b2f_nlmeans_dev: n_frames u8 frames [n][channels][height][width] in HBM -> d_out float [n][C][height][width] with
 *   C the mapped channel count, explicit parameters, no colour test.  One launch sequence for the whole batch,
 *   asynchronous on `stream` (NULL = ctx stream). */
int b2f_nlmeans_resolve(int channels, float sigma, int args_auto, int *win, int *bloc, float *filter);
int b2f_nlmeans_host_r32(b2f_ctx *ctx, const int32_t *image, int width, int height, int channels, float sigma, int args_auto,
                         int win, int bloc, float filter, float *out, int *out_channels, int *win_used, int *bloc_used,
                         float *filter_used);
int b2f_nlmeans_dev(b2f_ctx *ctx, const uint8_t *d_frames, int n_frames, int channels, int width, int height, int win, int bloc,
                    float sigma, float filter, float *d_out, void *stream);

/* ---------------------------------------------------------------------- face detection ----
 * The CNN face detector of image.libfacedetection (detect_faces, src/rcpp_libfacedetection.cpp, which calls facedetect_cnn
 * in facedetectcnn-model.cpp).  Detections are the reference's bit for bit, as gcc -O2 builds it on x86-64 (DESIGN.md §5).
 * The library ships no weights: the model is built from the R package's own table.
 * b2f_conv_layer: the layout of the reference's ConvInfoStruct, so its param_pConvInfo[24] can be passed as it is.
 *   weights are [num][channels][kernel_size][kernel_size].
 * b2f_facedet_model_create: checks the 24 layers against the network (shapes; stride 1 and pad 1 / 0 for the 3x3 / 1x1
 *   layers 1..23; layer 0 is 3x3 over 3 colours to 32 channels) and returns B2F_EINVAL with a message for anything else;
 *   repacks the weights once into device memory of ctx's device.  Released by b2f_facedet_model_free.
 * Faces are int32 [256][15] per frame: confidence, x, y, width, height, then the five landmark (x, y) pairs, after the
 *   reference's short casts; *n_faces (<= 100) of them are set, the rest are 0.
 * b2f_facedet_host_r32: the body of detect_faces.  x = x_len R integers, the interleaved RGB frame row by row (R's
 *   aperm(x, c(3, 2, 1))), narrowed like the glue's (unsigned char) cast.  step must be 3 * width and x_len at least
 *   3 * width * height (B2F_EINVAL otherwise); width or height <= 0 gives 0 faces, as in the reference.
 * b2f_facedet_batch_rgb: n_frames host frames [n][height][width][3] u8 -> n_faces [n], faces [n][256][15]; chunked, with the
 *   upload of the next chunk overlapping the current one.
 * b2f_facedet_dev: the same for frames in HBM, on `stream` (NULL = ctx stream); returns when the host outputs are written.
 *   Optional outputs: layer_max [n][16] = the per-frame maximum of each ReLU layer after the ReLU (-1 for a layer the
 *   reference does not run on a frame this small), and the candidate records the head pass sends to the host tail:
 *   cand [n][cand_cap][17] = (prior index in the reference's concatenation order, 2 conf ints, 14 loc ints) sorted by
 *   prior index, n_cand [n] = their number (records beyond cand_cap are counted but not written). */
typedef struct b2f_conv_layer {
  int pad, stride, kernel_size, channels, num;
  float scale;
  const int8_t *weights;
  const int32_t *bias;
} b2f_conv_layer;
typedef struct b2f_facedet_model b2f_facedet_model;
int b2f_facedet_model_create(b2f_ctx *ctx, const b2f_conv_layer *layers, int n_layers, b2f_facedet_model **model);
void b2f_facedet_model_free(b2f_facedet_model *model);
int b2f_facedet_host_r32(b2f_ctx *ctx, const b2f_facedet_model *model, const int32_t *x, size_t x_len, int width, int height,
                         int step, int *n_faces, int32_t *faces);
int b2f_facedet_batch_rgb(b2f_ctx *ctx, const b2f_facedet_model *model, const uint8_t *frames, int n_frames, int width, int height,
                          int *n_faces, int32_t *faces);
int b2f_facedet_dev(b2f_ctx *ctx, const b2f_facedet_model *model, const uint8_t *d_frames, int n_frames, int width, int height,
                    int *n_faces, int32_t *faces, int32_t *layer_max, int32_t *cand, int cand_cap, int *n_cand, void *stream);

/* ---------------------------------------------------------------------- darknet ----
 * YOLO detection and ImageNet classification of image.darknet (darknet_test_detector and darknet_predict_classifier),
 * bit-identical to the reference built with gcc -O2 on x86-64 (DESIGN.md §4.13, §5).  Convolutions sum in the reference's
 * exact order on the CUDA cores.  The library ships no weights: the model is built from a cfg and .weights file that the
 * caller parsed (image_b200/darknet.py, or the package's own parse_network_cfg + load_weights in the R glue).
 * b2f_darknet_layer: one cfg section.  type is B2F_DN_*; B2F_DN_OTHER (0) is a section the engine does not run, named
 *   by `name` in the error.  conv: filters, size, stride, pad (padding in pixels), batch_normalize, activation
 *   (B2F_DN_LINEAR / B2F_DN_LEAKY), biases [filters], scales / rolling_mean / rolling_variance [filters] when
 *   batch_normalize, weights [filters][c][size][size] with n_weights floats.  maxpool: size, stride, pad.  softmax:
 *   groups (must be 1), temperature.  region: classes, coords (must be 4), num, softmax, anchors [2 num].  tree != 0
 *   marks a softmax tree (unsupported).  avgpool and cost read no field.
 * b2f_darknet_model_create: checks the whole network at net_w x net_h (3 channels), and returns B2F_EINVAL with a message
 *   naming the layer for any unsupported layer or parameter (route, reorg, connected, dropout, crop, activations other
 *   than leaky / linear, softmax trees, a weights array shorter or longer than the layer needs).  Conv, maxpool and
 *   avgpool layers run on the GPU; softmax, region and cost may only follow them.  The weights go to ctx's device once.
 * b2f_darknet_model_dims: dims[0] = boxes per frame of the region layer (l.w * l.h * l.n, 0 without one), dims[1] = its
 *   classes, dims[2] = net.outputs (the length of the network output at net_w x net_h).
 * b2f_darknet_detect_*: frames [n][height][width][3] u8 -> per frame, after resize_image to net_w x net_h, the forward pass,
 *   get_region_boxes and do_nms_sort at nms .4: probs [n][boxes][classes + 1], boxes [n][boxes][4] (x, y, w, h) and
 *   count [n] = the boxes whose best class is above thresh.  hier_thresh only matters for softmax trees (not supported).
 * b2f_darknet_classify_*: resize_min(frame, net_w), the forward pass at that size (resize != 0) or at net_w x net_h on the
 *   first 3 net_w net_h floats of the resized planes (resize == 0), and top_k: index [n][top], prob [n][top].  top must be
 *   in 1..net.outputs.  The network may have no region layer.  With resize == 0, a frame whose resized planes hold fewer
 *   than net_w net_h pixels (a cfg taller than wide) gives B2F_EUNSUP: the reference reads past its buffer there.
 * The _batch_rgb forms take host frames (chunked, the upload of the next chunk overlapping the current one); the _dev forms
 *   frames in HBM, on `stream` (NULL = ctx stream), and return when the host outputs are written.
 * b2f_darknet_layer_dev: the output of layer `layer` (-1 = the network input: the resized planes) for mode 0 = detect,
 *   1 = classify with resize, 2 = classify without; out [n][c][h][w] floats with dims = (c, h, w).  out = NULL returns only
 *   dims; out_len must hold n c h w floats.  Region and softmax layers give the reference's l.output; cost layers are
 *   refused. */
enum { B2F_DN_OTHER = 0, B2F_DN_CONV = 1, B2F_DN_MAXPOOL = 2, B2F_DN_AVGPOOL = 3, B2F_DN_SOFTMAX = 4, B2F_DN_REGION = 5,
       B2F_DN_COST = 6 };
enum { B2F_DN_LINEAR = 0, B2F_DN_LEAKY = 1, B2F_DN_ACT_OTHER = 2 };
typedef struct b2f_darknet_layer {
  int type;
  const char *name;
  int filters, size, stride, pad, batch_normalize, activation;
  int groups;
  float temperature;
  int classes, coords, num, softmax, tree;
  const float *biases, *scales, *rolling_mean, *rolling_variance, *weights;
  size_t n_weights;
  const float *anchors;
} b2f_darknet_layer;
typedef struct b2f_darknet_model b2f_darknet_model;
int b2f_darknet_model_create(b2f_ctx *ctx, const b2f_darknet_layer *layers, int n_layers, int net_w, int net_h,
                             b2f_darknet_model **model);
void b2f_darknet_model_free(b2f_darknet_model *model);
int b2f_darknet_model_dims(const b2f_darknet_model *model, int *dims);
int b2f_darknet_detect_batch_rgb(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *frames, int n_frames, int width,
                                 int height, float thresh, float hier_thresh, float *probs, float *boxes, int *count);
int b2f_darknet_detect_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                           int height, float thresh, float hier_thresh, float *probs, float *boxes, int *count, void *stream);
int b2f_darknet_classify_batch_rgb(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *frames, int n_frames, int width,
                                   int height, int resize, int top, int *index, double *prob);
int b2f_darknet_classify_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                             int height, int resize, int top, int *index, double *prob, void *stream);
int b2f_darknet_layer_dev(b2f_ctx *ctx, const b2f_darknet_model *model, const uint8_t *d_frames, int n_frames, int width,
                          int height, int mode, int layer, float *out, size_t out_len, int *dims, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* B2F_H */
