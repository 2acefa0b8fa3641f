/* TEST INFRASTRUCTURE — C-callable layer driver around the UNMODIFIED reference functions of image.libfacedetection
 * (facedetectcnn.cpp, facedetectcnn-model.cpp), compiled in place into oracle/_ref/libref_facedetect.so together with
 * facedetectcnn-int8data.cpp.  facedetect_cnn itself is exported by the reference sources.
 *
 * ref_fd_run replays objectdetect_cnn (facedetectcnn-model.cpp:103-394) step by step with the reference's own
 * convolution_relu, maxpooling2x2S2, convolution, priorbox, blob2vector, convertInt2Float, concat4, softmax1vector2class and
 * detection_output, and keeps what the parity tests compare:
 *   - the nMax of each of the 16 ReLU layers (the maximum of the ReLU'd int32 plane, from the reference's convolution of
 *     the same input; -1 where the layer did not run), and the scale and bias of each ReLU output blob;
 *   - the eight head int32 planes and their scales;
 *   - the detections, and two counts: candidates above the confidence threshold, and boxes NMS keeps without the
 *     keep_top_k cut (a second detection_output call with keep_top_k = -1).
 * The ref_fd_* accessors copy them out.  Not thread-safe: one run at a time. */
#include <Rcpp.h>
#include <cstring>
#include <vector>
#include "facedetectcnn.h"

extern Filters g_pFilters[24];
extern bool param_initialized;
void init_parameters();

namespace {
struct Run {
  int nmax[16];
  float scale[16];
  int bias[16];
  std::vector<int> head[8];
  int head_dims[8][3];
  float head_scale[8];
  std::vector<float> faces;     // n x 15 floats as detection_output writes them
  std::vector<int> ints;        // n x 15 ints as objectdetect_cnn + facedetect_cnn convert them
  int n_above = 0, n_nms = 0;
} R;

int conv_max(CDataBlob<unsigned char> *in, const Filters *f) {
  CDataBlob<int> t;
  if (!convolution(in, f, &t)) return -1;
  int m = 0;
  for (int r = 0; r < t.height; r++)
    for (int c = 0; c < t.width; c++) {
      const int *p = t.data + (size_t(r) * t.width + c) * t.channelStep / sizeof(int);
      for (int ch = 0; ch < t.channels; ch++) m = MAX(MAX(p[ch], 0), m);
    }
  return m;
}
} // namespace

extern "C" {

int ref_fd_run(unsigned char *rgb, int width, int height, int step) {
  if (!param_initialized) { init_parameters(); param_initialized = true; }
  CDataBlob<unsigned char> input, relu[16], pool[5];
  CDataBlob<int> branch[8];
  input.setDataFrom3x3S2P1to1x1S1P0FromImage(rgb, width, height, 3, step);
  static const int pool_after[16] = {0, 1, 0, 2, 0, 0, 3, 0, 0, 4, 0, 0, 5, 0, 0, 0};
  CDataBlob<unsigned char> *cur = &input;
  for (int l = 0; l < 16; l++) {
    R.nmax[l] = cur->data ? conv_max(cur, g_pFilters + l) : -1;
    convolution_relu(cur, g_pFilters + l, relu + l);
    R.scale[l] = relu[l].scale;
    R.bias[l] = relu[l].bias;
    cur = relu + l;
    if (pool_after[l]) {
      maxpooling2x2S2(relu + l, pool + pool_after[l] - 1);
      cur = pool + pool_after[l] - 1;
    }
  }
  static const int src[4] = {6, 9, 12, 15};
  static const int nsz[4] = {3, 2, 2, 3}, stp[4] = {8, 16, 32, 64};
  static float sizes[4][3] = {{10, 16, 24}, {32, 48, 0}, {64, 96, 0}, {128, 192, 256}};
  CDataBlob<float> prior[4], prior_flat[4], loc_f[4], conf_f[4];
  CDataBlob<int> loc_flat[4], conf_flat[4];
  for (int h = 0; h < 4; h++) {
    for (int k = 0; k < 2; k++) {
      CDataBlob<int> &b = branch[2 * h + k];
      convolution(relu + src[h], g_pFilters + 16 + 2 * h + k, &b);
      R.head[2 * h + k].clear();
      R.head_dims[2 * h + k][0] = b.width; R.head_dims[2 * h + k][1] = b.height; R.head_dims[2 * h + k][2] = b.channels;
      R.head_scale[2 * h + k] = b.scale;
      if (b.data)
        for (int r = 0; r < b.height; r++)
          for (int c = 0; c < b.width; c++) {
            const int *p = b.data + (size_t(r) * b.width + c) * b.channelStep / sizeof(int);
            R.head[2 * h + k].insert(R.head[2 * h + k].end(), p, p + b.channels);
          }
    }
    priorbox(relu + src[h], width, height, stp[h], nsz[h], sizes[h], prior + h);
    blob2vector(prior + h, prior_flat + h);
    blob2vector(branch + 2 * h, loc_flat + h);
    blob2vector(branch + 2 * h + 1, conf_flat + h);
  }
  for (int h = 0; h < 4; h++) convertInt2Float(loc_flat + h, loc_f + h);
  for (int h = 0; h < 4; h++) convertInt2Float(conf_flat + h, conf_f + h);
  CDataBlob<float> mbox_prior, mbox_loc, mbox_conf, info, info_all;
  concat4(prior_flat, prior_flat + 1, prior_flat + 2, prior_flat + 3, &mbox_prior);
  concat4(loc_f, loc_f + 1, loc_f + 2, loc_f + 3, &mbox_loc);
  concat4(conf_f, conf_f + 1, conf_f + 2, conf_f + 3, &mbox_conf);
  softmax1vector2class(&mbox_conf);
  R.n_above = 0;
  if (mbox_conf.data && mbox_conf.width == 1 && mbox_conf.height == 1)
    for (int i = 0; i < mbox_conf.channels; i += 2) R.n_above += mbox_conf.data[i + 1] > 0.5f;
  detection_output(&mbox_prior, &mbox_loc, &mbox_conf, 0.3f, 0.5f, 1000, 100, &info);
  detection_output(&mbox_prior, &mbox_loc, &mbox_conf, 0.3f, 0.5f, 1000, -1, &info_all);
  R.n_nms = info_all.width;
  R.faces.clear();
  R.ints.clear();
  for (int i = 0; i < info.width; i++) {       // objectdetect_cnn's conversion, then facedetect_cnn's short casts
    float v[15];
    for (int k = 0; k < 15; k++) v[k] = info.getElement(i, 0, k);
    R.faces.insert(R.faces.end(), v, v + 15);
    FaceRect r;
    r.score = v[0];
    r.x = int(v[1] * width + 0.5f);
    r.y = int(v[2] * height + 0.5f);
    r.w = int((v[3] - v[1]) * width + 0.5f);
    r.h = int((v[4] - v[2]) * height + 0.5f);
    for (int lm = 0; lm < 5; lm++) {
      r.lm[lm * 2] = int(v[5 + lm * 2] * width + 0.5f);
      r.lm[lm * 2 + 1] = int(v[5 + lm * 2 + 1] * height + 0.5f);
    }
    short p[15];
    p[0] = (short)(r.score * r.score * 100);
    p[1] = (short)r.x; p[2] = (short)r.y; p[3] = (short)r.w; p[4] = (short)r.h;
    for (int lm = 0; lm < 10; lm++) p[5 + lm] = (short)r.lm[lm];
    R.ints.insert(R.ints.end(), p, p + 15);
  }
  return info.width;
}

void ref_fd_trunk(int *nmax, float *scale, int *bias) {
  std::memcpy(nmax, R.nmax, sizeof R.nmax);
  std::memcpy(scale, R.scale, sizeof R.scale);
  std::memcpy(bias, R.bias, sizeof R.bias);
}

/* dims = (width, height, channels) of head k (0..7: L16..L23); copies the plane when out != NULL */
void ref_fd_head(int k, int *dims, float *scale, int *out) {
  std::memcpy(dims, R.head_dims[k], 3 * sizeof(int));
  *scale = R.head_scale[k];
  if (out && !R.head[k].empty()) std::memcpy(out, R.head[k].data(), R.head[k].size() * sizeof(int));
}

void ref_fd_faces(float *f, int *ints) {
  if (!R.faces.empty()) std::memcpy(f, R.faces.data(), R.faces.size() * sizeof(float));
  if (!R.ints.empty()) std::memcpy(ints, R.ints.data(), R.ints.size() * sizeof(int));
}

void ref_fd_counts(int *n_above, int *n_nms) { *n_above = R.n_above; *n_nms = R.n_nms; }

/* facedetect_cnn (facedetectcnn-model.cpp:395-437) as detect_faces calls it: returns the face count and copies the 15
 * shorts of each face into faces[n][15] as ints */
int ref_facedetect_cnn(unsigned char *rgb, int width, int height, int step, int *faces) {
  std::vector<unsigned char> buf(0x20000);
  int *r = facedetect_cnn(buf.data(), rgb, width, height, step);
  const int n = r ? *r : 0;
  for (int i = 0; i < n; i++) {
    const short *p = ((const short *)(r + 1)) + 142 * i;
    for (int k = 0; k < 15; k++) faces[i * 15 + k] = p[k];
  }
  return n;
}

} // extern "C"
