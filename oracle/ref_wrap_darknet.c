/* TEST INFRASTRUCTURE.  A driver over the reference build of image.darknet (oracle/darknet.mk): one network at a time,
 * parsed and loaded by the reference's own parse_network_cfg + load_weights, run by its own network_predict, with the
 * detection tail of darknet_test_detector (get_region_boxes, do_nms_sort at nms .4, the count above the threshold) and
 * the classifier tail of darknet_predict_classifier (resize_min, resize_network, top_k).  Frames come in as interleaved
 * u8 RGB and become the reference's planar floats as load_image_stb does it; ref_dn_decode decodes a file with the
 * reference's own stb_image.  Everything is batch 1, as the R glue runs it. */
#include <stdlib.h>
#include <string.h>

#include "box.h"
#include "image.h"
#include "layer.h"
#include "network.h"
#include "parser.h"
#include "region_layer.h"
#include "stb_image.h"
#include "utils.h"

static network net;
static int have_net = 0, cfg_w = 0, cfg_h = 0;

int ref_dn_load(char *cfg, char *weights) {
  if (have_net) free_network(net);
  net = parse_network_cfg(cfg);
  if (weights && weights[0]) load_weights(&net, weights);
  set_batch_network(&net, 1);
  have_net = 1;
  cfg_w = net.w;
  cfg_h = net.h;
  return net.n;
}

/* u8 RGB of a file, decoded by the reference's stbi_load(.., 3): returns 0 and w, h only when out is NULL. */
int ref_dn_decode(const char *file, int *w, int *h, unsigned char *out) {
  int c;
  unsigned char *d = stbi_load(file, w, h, &c, 3);
  if (!d) return -1;
  if (out) memcpy(out, d, (size_t)(*w) * (*h) * 3);
  free(d);
  return 0;
}

/* load_image_stb's conversion of an interleaved u8 frame */
static image to_image(const unsigned char *rgb, int w, int h) {
  image im = make_image(w, h, 3);
  int i, j, k;
  for (k = 0; k < 3; ++k)
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) im.data[i + w * j + w * h * k] = (float)rgb[k + 3 * i + 3 * w * j] / 255.;
  return im;
}

/* The network input a frame becomes: mode 0 = detect (resize_image to the cfg size), 1 = classify with resize,
 * 2 = classify without resize.  Writes the planar floats when out != NULL and returns their count; *nw, *nh are the
 * network size the forward pass runs at. */
static image net_input(const unsigned char *rgb, int w, int h, int mode, int *nw, int *nh, image *orig) {
  image im = to_image(rgb, w, h), r;
  if (mode == 0) {
    r = resize_image(im, cfg_w, cfg_h);
    *nw = cfg_w; *nh = cfg_h;
  } else {
    r = resize_min(im, cfg_w);
    if (mode == 1) { *nw = r.w; *nh = r.h; } else { *nw = cfg_w; *nh = cfg_h; }
  }
  *orig = im;
  return r;
}

int ref_dn_input(const unsigned char *rgb, int w, int h, int mode, float *out, int *dims) {
  int nw, nh;
  image im, r = net_input(rgb, w, h, mode, &nw, &nh, &im);
  int n = r.w * r.h * 3;
  if (out) memcpy(out, r.data, (size_t)n * sizeof(float));
  dims[0] = 3; dims[1] = r.h; dims[2] = r.w;
  if (r.data != im.data) free_image(r);
  free_image(im);
  return n;
}

/* network_predict of one frame; the layer outputs stay in the network until the next call. */
int ref_dn_forward(const unsigned char *rgb, int w, int h, int mode) {
  int nw, nh;
  image im, r = net_input(rgb, w, h, mode, &nw, &nh, &im);
  if (net.w != nw || net.h != nh) resize_network(&net, nw, nh);
  network_predict(net, r.data);
  if (r.data != im.data) free_image(r);
  free_image(im);
  return 0;
}

/* Layer i: info = type, c, h, w, out_c, out_h, out_w, n, size, stride, pad, batch_normalize, activation, outputs,
 * classes, coords, softmax, groups.  Its output of the last forward pass goes to out when out != NULL. */
int ref_dn_layer(int i, int *info, float *out) {
  layer l = net.layers[i];
  int v[18] = {l.type, l.c, l.h, l.w, l.out_c, l.out_h, l.out_w, l.n, l.size, l.stride, l.pad, l.batch_normalize,
               l.activation, l.outputs, l.classes, l.coords, l.softmax, l.groups};
  memcpy(info, v, sizeof(v));
  if (out && l.output) memcpy(out, l.output, (size_t)l.outputs * sizeof(float));
  return l.outputs;
}

/* The parameter arrays of layer i as load_weights left them (NULL pointers are skipped). */
void ref_dn_params(int i, float *biases, float *scales, float *mean, float *var, float *weights, float *anchors) {
  layer l = net.layers[i];
  if (l.type == CONVOLUTIONAL) {
    memcpy(biases, l.biases, l.n * sizeof(float));
    if (l.batch_normalize && scales) {
      memcpy(scales, l.scales, l.n * sizeof(float));
      memcpy(mean, l.rolling_mean, l.n * sizeof(float));
      memcpy(var, l.rolling_variance, l.n * sizeof(float));
    }
    memcpy(weights, l.weights, (size_t)l.n * l.c * l.size * l.size * sizeof(float));
  } else if (l.type == REGION && anchors) {
    memcpy(anchors, l.biases, 2 * l.n * sizeof(float));
  }
}

/* darknet_test_detector without drawing: probs [total][classes + 1] and boxes [total][4] after NMS; returns the count
 * above the threshold. */
int ref_dn_detect(const unsigned char *rgb, int w, int h, float thresh, float hier_thresh, float *probs_out, float *boxes_out) {
  ref_dn_forward(rgb, w, h, 0);
  layer l = net.layers[net.n - 1];
  int total = l.w * l.h * l.n, j, found = 0;
  float nms = .4;
  box *boxes = calloc(total, sizeof(box));
  float **probs = calloc(total, sizeof(float *));
  for (j = 0; j < total; ++j) probs[j] = calloc(l.classes + 1, sizeof(float *));
  get_region_boxes(l, 1, 1, thresh, probs, boxes, 0, 0, hier_thresh);
  if (l.softmax_tree && nms) do_nms_obj(boxes, probs, total, l.classes, nms);
  else if (nms) do_nms_sort(boxes, probs, total, l.classes, nms);
  for (j = 0; j < total; ++j) {
    int cls = max_index(probs[j], l.classes);
    if (probs[j][cls] > thresh) found++;
    memcpy(probs_out + (size_t)j * (l.classes + 1), probs[j], (l.classes + 1) * sizeof(float));
    boxes_out[4 * j + 0] = boxes[j].x; boxes_out[4 * j + 1] = boxes[j].y;
    boxes_out[4 * j + 2] = boxes[j].w; boxes_out[4 * j + 3] = boxes[j].h;
  }
  free(boxes);
  free_ptrs((void **)probs, total);
  return found;
}

/* darknet_predict_classifier: top indices and their probabilities (as the doubles R gets), and the whole output vector
 * when pred != NULL.  Returns net.outputs. */
int ref_dn_classify(const unsigned char *rgb, int w, int h, int resize, int top, int *idx, double *score, float *pred) {
  if (!resize && (net.w != cfg_w || net.h != cfg_h)) resize_network(&net, cfg_w, cfg_h);
  ref_dn_forward(rgb, w, h, resize ? 1 : 2);
  float *p = get_network_output(net);
  int i;
  top_k(p, net.outputs, top, idx);
  for (i = 0; i < top; ++i) score[i] = p[idx[i]];
  if (pred) memcpy(pred, p, (size_t)net.outputs * sizeof(float));
  return net.outputs;
}

int ref_dn_net(int *info) {
  info[0] = net.n; info[1] = cfg_w; info[2] = cfg_h; info[3] = net.c; info[4] = net.outputs;
  return net.n;
}
