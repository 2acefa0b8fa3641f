/* TEST INFRASTRUCTURE — the mock Rcpp of oracle/stubs plus the one conversion the glue of image.DenoiseNLMeans
 * (src/rcpp_denoisenlmeans.cpp) needs: Rcpp::as<std::vector<float> >(IntegerVector), an element-wise static_cast as Rcpp's
 * container conversion does.  Put this directory before oracle/stubs on the include path.  Not Rcpp, not product code. */
#ifndef ORACLE_STUB_RCPP_NLMEANS_H
#define ORACLE_STUB_RCPP_NLMEANS_H
#include "../stubs/Rcpp.h"

namespace Rcpp {
template <typename T, typename S> T as(const VecT<S> &v) { return T(v.d.begin(), v.d.end()); }
} // namespace Rcpp
#endif
