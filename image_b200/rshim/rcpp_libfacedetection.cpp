// Replacement body for detect_faces (image.libfacedetection/src/rcpp_libfacedetection.cpp) — same exported signature, same
// return list.  The package keeps facedetectcnn-int8data.cpp for its weight table, param_pConvInfo, whose ConvInfoStruct
// layout is b2f_conv_layer's; the model is built from it once per R session.
#include <Rcpp.h>
#include <Rcpp/DataFrame.h>      // already part of <Rcpp.h>; named for the DataFrame::create below
#include <vector>
#include "b2f_r_context.h"

extern b2f_conv_layer param_pConvInfo[24];   // facedetectcnn-int8data.cpp (ConvInfoStruct, the same layout)

static b2f_facedet_model *b2f_r_facedet_model() {
  static b2f_facedet_model *m = nullptr;
  if (!m) b2f_r_check(b2f_facedet_model_create(b2f_r_ctx(), param_pConvInfo, 24, &m));
  return m;
}

// [[Rcpp::export]]
Rcpp::List detect_faces(Rcpp::IntegerVector x, int width, int height, int step) {
  int nr = 0;
  std::vector<int32_t> f(256 * 15);
  b2f_r_check(b2f_facedet_host_r32(b2f_r_ctx(), b2f_r_facedet_model(), x.size() ? &x[0] : nullptr, (size_t)x.size(), width, height,
                                   step, &nr, f.data()));
  std::vector<int> col[15];
  for (int i = 0; i < nr; i++)
    for (int k = 0; k < 15; k++) col[k].push_back(f[i * 15 + k]);
  return Rcpp::List::create(
      Rcpp::Named("nr") = nr,
      Rcpp::Named("detections") = Rcpp::DataFrame::create(
          Rcpp::Named("x") = col[1], Rcpp::Named("y") = col[2], Rcpp::Named("width") = col[3], Rcpp::Named("height") = col[4],
          Rcpp::Named("confidence") = col[0], Rcpp::Named("landmark1_x") = col[5], Rcpp::Named("landmark1_y") = col[6],
          Rcpp::Named("landmark2_x") = col[7], Rcpp::Named("landmark2_y") = col[8], Rcpp::Named("landmark3_x") = col[9],
          Rcpp::Named("landmark3_y") = col[10], Rcpp::Named("landmark4_x") = col[11], Rcpp::Named("landmark4_y") = col[12],
          Rcpp::Named("landmark5_x") = col[13], Rcpp::Named("landmark5_y") = col[14]));
}
