/* TEST INFRASTRUCTURE — mock of Rcpp's <Rcpp/DataFrame.h> for the mock Rcpp of ../Rcpp.h: DataFrame::create of equally long
 * Named columns, as image.libfacedetection/src/rcpp_libfacedetection.cpp:81-99 builds its `detections`.  The frame is
 * held as an nr x nc NumericMatrix, column after column (the mock's Named(...) = matrix keeps nr and nc); the column
 * names are not kept.  Not Rcpp, not product code. */
#ifndef ORACLE_STUB_RCPP_DATAFRAME_H
#define ORACLE_STUB_RCPP_DATAFRAME_H
#include <initializer_list>
#include <stdexcept>
#include <vector>
#include "../Rcpp.h"

namespace Rcpp {
struct DataFrame {
  template <typename... A> static NumericMatrix create(const A &... a) {
    std::vector<Value> cols;
    (void)std::initializer_list<int>{(cols.push_back(a), 0)...};
    const long nr = cols.empty() ? 0 : (long)cols[0].data.size();
    NumericMatrix m(nr, (long)cols.size());
    for (size_t j = 0; j < cols.size(); j++) {
      if ((long)cols[j].data.size() != nr) throw std::runtime_error("DataFrame::create: columns of different lengths");
      for (long i = 0; i < nr; i++) m((long)i, (long)j) = cols[j].data[(size_t)i];
    }
    return m;
  }
};
} // namespace Rcpp
#endif
