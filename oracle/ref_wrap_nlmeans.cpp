/* TEST INFRASTRUCTURE — C-callable wrapper around the UNMODIFIED reference entry point rcpp_nlmeans()
 * (image.DenoiseNLMeans/src/rcpp_denoisenlmeans.cpp), compiled in place together with libdenoising.cpp,
 * libauxiliar.cpp and mt19937ar.c into oracle/_ref/libref_nlmeans.so, WITHOUT -fopenmp: the reference's parallel
 * loop races on its output rows, and the serial order is the contract (DESIGN.md §5). */
#include <Rcpp.h>
#include <cstring>

Rcpp::List rcpp_nlmeans(Rcpp::IntegerVector image, int width, int height, int channels, float sigma, bool args_auto,
                        int win, int bloc, float fFiltPar);

extern "C" {

/* image = width*height*channels ints.  out receives the `denoised` doubles (room for width*height*3).  Returns 0, or -1
 * with the Rcpp::stop message in err. */
int ref_nlmeans(const int *image, int width, int height, int channels, float sigma, int args_auto, int win, int bloc,
                float filter, double *out, int *out_channels, int *win_used, int *bloc_used, float *filter_used,
                float *sigma_used, char *err, int errcap) {
  try {
    Rcpp::IntegerVector v(image, (size_t)width * height * channels);
    Rcpp::List l = rcpp_nlmeans(v, width, height, channels, sigma, args_auto != 0, win, bloc, filter);
    const std::vector<double> &d = l.get("denoised").data;
    for (size_t i = 0; i < d.size(); i++) out[i] = d[i];
    *out_channels = (int)l.get("channels").data[0];
    *win_used = (int)l.get("window").data[0];
    *bloc_used = (int)l.get("bloc").data[0];
    *filter_used = (float)l.get("filter").data[0];
    *sigma_used = (float)l.get("sigma").data[0];
    return 0;
  } catch (std::exception &e) {
    if (err && errcap > 0) { std::strncpy(err, e.what(), (size_t)errcap - 1); err[errcap - 1] = 0; }
    return -1;
  }
}

} // extern "C"
