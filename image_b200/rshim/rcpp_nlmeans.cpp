// Replacement body for rcpp_nlmeans (image.DenoiseNLMeans/src/rcpp_denoisenlmeans.cpp) — same exported signature, same
// return list.  Narrowing, the colour test, the parameter table and the denoising run behind the C ABI of include/b2f.h.
#include <Rcpp.h>
#include <vector>
#include "b2f_r_context.h"

// [[Rcpp::plugins(cpp11)]]
// [[Rcpp::export]]
Rcpp::List rcpp_nlmeans(Rcpp::IntegerVector image, int width, int height, int channels, float sigma, bool args_auto = true,
                        int win = 1, int bloc = 10, float fFiltPar = 0.4) {
  if (width <= 0 || height <= 0 || channels <= 0) Rcpp::stop("rcpp_nlmeans: width, height and channels must be positive");
  const size_t n = (size_t)width * height;
  // (the reference reads past the end of a shorter vector)
  if ((size_t)image.size() < n * (size_t)channels) Rcpp::stop("rcpp_nlmeans: image must hold width*height*channels values");
  std::vector<float> out(n * (channels == 2 ? 1 : channels > 3 ? 3 : channels));
  int d_c = 0, w = 0, b = 0;
  float filter = 0.0f;
  if (b2f_nlmeans_host_r32(b2f_r_ctx(), &image[0], width, height, channels, sigma, args_auto ? 1 : 0, win, bloc, fFiltPar,
                           out.data(), &d_c, &w, &b, &filter) != B2F_OK)
    Rcpp::stop(b2f_last_error());                      // the table's message is the reference's own
  std::vector<double> denoised(out.begin(), out.begin() + n * d_c);
  return Rcpp::List::create(Rcpp::Named("width") = width, Rcpp::Named("height") = height, Rcpp::Named("channels") = d_c,
                            Rcpp::Named("denoised") = denoised, Rcpp::Named("sigma") = sigma, Rcpp::Named("filter") = filter,
                            Rcpp::Named("window") = w, Rcpp::Named("bloc") = b);
}
