/* darknet_r_api.c — replaces image.darknet's src/__R_API_detector.c and src/__R_API_classifier.c.  The .Call entry
 * points darknet_detect and darknet_predict and the bodies darknet_test_detector / darknet_predict_classifier keep
 * their signatures, the package's own parse_network_cfg + load_weights, the frame decode by stbi_load(.., 3), the
 * printed lines, draw_detections + save_image and the return values.  Only the forward pass and the tails that read
 * the network output move to libb200feat: resize_image + network_predict + get_region_boxes + do_nms_sort become
 * b2f_darknet_detect_batch_rgb, and resize_min + network_predict + top_k become b2f_darknet_classify_batch_rgb, whose
 * results are the reference's bit for bit (DESIGN.md §4.13, §5).  A network the engine does not run (route, reorg,
 * connected, ... layers: b2f_darknet_model_create returns B2F_EINVAL) keeps the reference's own forward pass. */
#include "network.h"
#include "region_layer.h"
#include "cost_layer.h"
#include "utils.h"
#include "parser.h"
#include "box.h"
#include "image.h"
#include "stb_image.h"

#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "b2f.h"

#include <R.h>
#include <Rinternals.h>
#include <Rdefines.h>

/* one libb200feat context per R session (R calls .Call from its main thread only) */
static b2f_ctx *b2f_dn_ctx(void) {
  static b2f_ctx *ctx = NULL;
  if (!ctx) {
    const char *e = getenv("B2F_DEVICE");
    if (b2f_init(e ? atoi(e) : 0, &ctx) != B2F_OK) Rf_error("libb200feat: %s", b2f_last_error());
  }
  return ctx;
}

static const char *b2f_dn_name(LAYER_TYPE t) {
  switch (t) {
    case ROUTE: return "route";
    case REORG: return "reorg";
    case CONNECTED: return "connected";
    case DROPOUT: return "dropout";
    case CROP: return "crop";
    case ACTIVE: return "activation";
    case SHORTCUT: return "shortcut";
    case NORMALIZATION: return "normalization";
    case BATCHNORM: return "batchnorm";
    case DETECTION: return "detection";
    case LOCAL: return "local";
    default: return "layer";
  }
}

/* The engine's model of a parsed and loaded network; B2F_EINVAL when it has a layer the engine does not run. */
static int b2f_dn_model(network *net, b2f_darknet_model **model) {
  b2f_darknet_layer *d = calloc(net->n, sizeof(b2f_darknet_layer));
  int i, rc;
  for (i = 0; i < net->n; ++i) {
    layer *l = &net->layers[i];
    b2f_darknet_layer *o = &d[i];
    o->name = b2f_dn_name(l->type);
    if (l->type == CONVOLUTIONAL) {
      o->type = B2F_DN_CONV;
      o->name = "convolutional";
      o->filters = l->n; o->size = l->size; o->stride = l->stride; o->pad = l->pad;
      o->batch_normalize = l->batch_normalize;
      o->activation = l->binary || l->xnor ? B2F_DN_ACT_OTHER
                      : l->activation == LEAKY ? B2F_DN_LEAKY : l->activation == LINEAR ? B2F_DN_LINEAR : B2F_DN_ACT_OTHER;
      o->biases = l->biases; o->scales = l->scales; o->rolling_mean = l->rolling_mean;
      o->rolling_variance = l->rolling_variance; o->weights = l->weights;
      o->n_weights = (size_t)l->n * l->c * l->size * l->size;
    } else if (l->type == MAXPOOL) {
      o->type = B2F_DN_MAXPOOL; o->name = "maxpool";
      o->size = l->size; o->stride = l->stride; o->pad = l->pad;
    } else if (l->type == AVGPOOL) {
      o->type = B2F_DN_AVGPOOL; o->name = "avgpool";
    } else if (l->type == SOFTMAX) {
      o->type = B2F_DN_SOFTMAX; o->name = "softmax";
      o->groups = l->groups; o->temperature = l->temperature; o->tree = l->softmax_tree != 0;
    } else if (l->type == REGION) {
      o->type = B2F_DN_REGION; o->name = "region";
      o->classes = l->classes; o->coords = l->coords; o->num = l->n; o->softmax = l->softmax;
      o->tree = l->softmax_tree != 0; o->anchors = l->biases;
    } else if (l->type == COST) {
      o->type = B2F_DN_COST; o->name = "cost";
    } else {
      o->type = B2F_DN_OTHER;
    }
  }
  rc = b2f_darknet_model_create(b2f_dn_ctx(), d, net->n, net->w, net->h, model);
  free(d);
  if (rc != B2F_OK && rc != B2F_EINVAL) Rf_error("libb200feat: %s", b2f_last_error());
  return rc;
}

/* the frame as bytes (stbi_load(.., 3)) and as the package's planar image, converted as load_image_stb does it; a file
 * stbi cannot read goes through load_image_color, which prints the reference's message */
static unsigned char *b2f_dn_load(char *filename, image *im) {
  int w, h, c, i, j, k;
  unsigned char *data = stbi_load(filename, &w, &h, &c, 3);
  if (!data) {
    *im = load_image_color(filename, 0, 0);
    return NULL;
  }
  *im = make_image(w, h, 3);
  for (k = 0; k < 3; ++k)
    for (j = 0; j < h; ++j)
      for (i = 0; i < w; ++i) im->data[i + w * j + w * h * k] = (float)data[k + 3 * i + 3 * w * j] / 255.;
  return data;
}

image **load_alphabet_pkg(char *path) {
  const int nsize = 8;
  int i, j;
  image **alphabets = calloc(nsize, sizeof(image));
  for (j = 0; j < nsize; ++j) {
    alphabets[j] = calloc(128, sizeof(image));
    for (i = 32; i < 127; ++i) {
      char buff[256];
      sprintf(buff, "%s/data/labels/%d_%d.png", path, i, j);
      alphabets[j][i] = load_image_color(buff, 0, 0);
    }
  }
  return alphabets;
}

int darknet_test_detector(char *cfgfile, char *weightfile, char *filename, float thresh, float hier_thresh, char **names, char *path) {
  image **alphabet = load_alphabet_pkg(path);
  network net = parse_network_cfg(cfgfile);
  if (weightfile) load_weights(&net, weightfile);
  set_batch_network(&net, 1);
  srand(2222222);
  char buff[256];
  char *input = buff;
  int j, found = 0;
  float nms = .4;
  b2f_darknet_model *model = NULL;
  const int on_gpu = b2f_dn_model(&net, &model) == B2F_OK;
  strncpy(input, filename, 256);
  image im;
  unsigned char *bytes = b2f_dn_load(input, &im);
  layer l = net.layers[net.n - 1];
  const int total = l.w * l.h * l.n;
  box *boxes = calloc(total, sizeof(box));
  float **probs = calloc(total, sizeof(float *));
  for (j = 0; j < total; ++j) probs[j] = calloc(l.classes + 1, sizeof(float *));
  clock_t time = clock();
  if (on_gpu) {
    float *p = malloc(sizeof(float) * total * (l.classes + 1)), *b = malloc(sizeof(float) * total * 4);
    int rc = b2f_darknet_detect_batch_rgb(b2f_dn_ctx(), model, bytes, 1, im.w, im.h, thresh, hier_thresh, p, b, &found);
    b2f_darknet_model_free(model);
    if (rc != B2F_OK) Rf_error("libb200feat: %s", b2f_last_error());
    printf("%s: Predicted in %f seconds.\n", input, sec(clock() - time));
    for (j = 0; j < total; ++j) {
      memcpy(probs[j], p + (size_t)j * (l.classes + 1), sizeof(float) * (l.classes + 1));
      boxes[j].x = b[4 * j]; boxes[j].y = b[4 * j + 1]; boxes[j].w = b[4 * j + 2]; boxes[j].h = b[4 * j + 3];
    }
    free(p);
    free(b);
  } else {
    image sized = resize_image(im, net.w, net.h);
    network_predict(net, sized.data);
    printf("%s: Predicted in %f seconds.\n", input, sec(clock() - time));
    get_region_boxes(l, 1, 1, thresh, probs, boxes, 0, 0, hier_thresh);
    if (l.softmax_tree && nms) do_nms_obj(boxes, probs, total, l.classes, nms);
    else if (nms) do_nms_sort(boxes, probs, total, l.classes, nms);
    for (j = 0; j < total; ++j) {
      int cls = max_index(probs[j], l.classes);
      if (probs[j][cls] > thresh) found++;
    }
    free_image(sized);
  }
  printf("Boxes: %d of which %d above the threshold.\n", total, found);
  draw_detections(im, total, thresh, boxes, probs, names, alphabet, l.classes);
  save_image(im, "predictions");
  free_image(im);
  free(bytes);
  free(boxes);
  free_ptrs((void **)probs, total);
  return found;
}

SEXP darknet_detect(SEXP modelsetup, SEXP modelweights, SEXP image_file, SEXP th, SEXP hier_th, SEXP labels, SEXP darknet_root) {
  const char *cfgfile = CHAR(STRING_ELT(modelsetup, 0));
  const char *weightfile = CHAR(STRING_ELT(modelweights, 0));
  const char *filename = CHAR(STRING_ELT(image_file, 0));
  const char *path = CHAR(STRING_ELT(darknet_root, 0));
  PROTECT(labels = AS_CHARACTER(labels));
  int i, n = LENGTH(labels);
  char **names = malloc(sizeof(char *) * (n > 0 ? n : 1));
  for (i = 0; i < n; i++) names[i] = (char *)CHAR(STRING_ELT(labels, i));
  darknet_test_detector((char *)cfgfile, (char *)weightfile, (char *)filename, REAL(th)[0], REAL(hier_th)[0], names, (char *)path);
  free(names);
  UNPROTECT(1);
  return modelsetup;
}

void darknet_predict_classifier(char *datacfg, char *cfgfile, char *weightfile, char *filename, int top, char **pred_lab,
                                double *pred_score, char **names, int resize) {
  network net = parse_network_cfg(cfgfile);
  if (weightfile) load_weights(&net, weightfile);
  set_batch_network(&net, 1);
  srand(2222222);
  (void)datacfg;
  char buff[256];
  char *input = buff;
  int i;
  int *indexes = calloc(top > 0 ? top : 1, sizeof(int));
  b2f_darknet_model *model = NULL;
  const int on_gpu = b2f_dn_model(&net, &model) == B2F_OK;
  strncpy(input, filename, 256);
  image im;
  unsigned char *bytes = b2f_dn_load(input, &im);
  if (on_gpu) {
    double *score = calloc(top > 0 ? top : 1, sizeof(double));
    int rc = b2f_darknet_classify_batch_rgb(b2f_dn_ctx(), model, bytes, 1, im.w, im.h, resize > 0, top, indexes, score);
    b2f_darknet_model_free(model);
    if (rc != B2F_OK) Rf_error("libb200feat: %s", b2f_last_error());
    for (i = 0; i < top; ++i) {
      pred_lab[i] = names[indexes[i]];
      pred_score[i] = score[i];
    }
    free(score);
  } else {
    image r = resize_min(im, net.w);
    if (resize > 0) resize_network(&net, r.w, r.h);
    float *predictions = network_predict(net, r.data);
    if (net.hierarchy) hierarchy_predictions(predictions, net.outputs, net.hierarchy, 0);
    top_k(predictions, net.outputs, top, indexes);
    for (i = 0; i < top; ++i) {
      pred_lab[i] = names[indexes[i]];
      pred_score[i] = predictions[indexes[i]];
    }
    if (r.data != im.data) free_image(r);
  }
  free_image(im);
  free(bytes);
  free(indexes);
}

SEXP darknet_predict(SEXP datasetup, SEXP modelsetup, SEXP modelweights, SEXP image_file, SEXP first, SEXP labels, SEXP resize) {
  const char *datacfg = CHAR(STRING_ELT(datasetup, 0));
  const char *cfgfile = CHAR(STRING_ELT(modelsetup, 0));
  const char *weightfile = CHAR(STRING_ELT(modelweights, 0));
  const char *filename = CHAR(STRING_ELT(image_file, 0));
  int top = INTEGER(first)[0];
  int i, n;
  char **pred_lab = malloc(sizeof(char *) * (top > 0 ? top : 1));
  double *pred_score = malloc(sizeof(double) * (top > 0 ? top : 1));
  PROTECT(labels = AS_CHARACTER(labels));
  n = LENGTH(labels);
  char **names = malloc(sizeof(char *) * (n > 0 ? n : 1));
  for (i = 0; i < n; i++) names[i] = (char *)CHAR(STRING_ELT(labels, i));
  darknet_predict_classifier((char *)datacfg, (char *)cfgfile, (char *)weightfile, (char *)filename, top, pred_lab, pred_score,
                             names, INTEGER(resize)[0]);
  SEXP labs = PROTECT(allocVector(STRSXP, top));
  SEXP scores = PROTECT(allocVector(REALSXP, top));
  SEXP result = PROTECT(allocVector(VECSXP, 2));
  SET_VECTOR_ELT(result, 0, scores);
  SET_VECTOR_ELT(result, 1, labs);
  for (i = 0; i < top; ++i) {
    SET_STRING_ELT(labs, i, mkChar(pred_lab[i]));
    REAL(scores)[i] = pred_score[i];
  }
  free(names);
  free(pred_lab);
  free(pred_score);
  UNPROTECT(4);
  return result;
}
