/* TEST INFRASTRUCTURE — the two names the sources of image.libfacedetection (facedetectcnn.cpp, facedetectcnn-model.cpp,
 * facedetectcnn-int8data.cpp) take from Rcpp: the Rcerr stream and REprintf.  Both write to stderr.  Not Rcpp, not
 * product code. */
#ifndef ORACLE_STUB_RCPP_FACEDETECT_H
#define ORACLE_STUB_RCPP_FACEDETECT_H
#include <cstdio>
#include <iostream>

namespace Rcpp {
static std::ostream &Rcerr = std::cerr;
} // namespace Rcpp
#define REprintf(...) std::fprintf(stderr, __VA_ARGS__)
#endif
