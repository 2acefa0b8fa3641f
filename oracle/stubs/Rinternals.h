/* TEST INFRASTRUCTURE — minimal stand-in for R's <Rinternals.h>, used only to compile R glue written in C (the
 * reference's image.darknet/src/__R_API_*.c and image_b200/rshim/darknet_r_api.c) into test programs: R is not
 * installed here.  A SEXP is a tagged vector of doubles, ints, strings (CHARSXP elements) or SEXPs, allocated with
 * malloc and never freed (a test program makes a handful).  Only the names that glue uses are provided. */
#ifndef ORACLE_STUB_RINTERNALS_H
#define ORACLE_STUB_RINTERNALS_H
#include <stdlib.h>
#include <string.h>
#include "R.h"
#ifdef __cplusplus
extern "C" {
#endif
enum { CHARSXP = 9, INTSXP = 13, REALSXP = 14, STRSXP = 16, VECSXP = 19 };
typedef struct stub_sexp *SEXP;
struct stub_sexp {
  int type;
  int length;
  void *data;   /* double[] / int[] / SEXP[] / char[] */
};
static inline SEXP Rf_allocVector(int type, int n) {
  SEXP s = (SEXP)calloc(1, sizeof(*s));
  size_t el = type == REALSXP ? sizeof(double) : type == INTSXP ? sizeof(int) : type == CHARSXP ? 1 : sizeof(SEXP);
  s->type = type;
  s->length = n;
  s->data = calloc((size_t)n + 1, el);
  return s;
}
static inline SEXP Rf_mkChar(const char *c) {
  SEXP s = Rf_allocVector(CHARSXP, (int)strlen(c));
  memcpy(s->data, c, strlen(c));
  return s;
}
#define allocVector Rf_allocVector
#define mkChar Rf_mkChar
#define PROTECT(x) (x)
#define UNPROTECT(n) ((void)(n))
#define LENGTH(x) ((x)->length)
#define REAL(x) ((double *)(x)->data)
#define INTEGER(x) ((int *)(x)->data)
#define CHAR(x) ((const char *)(x)->data)
#define STRING_ELT(x, i) (((SEXP *)(x)->data)[i])
#define VECTOR_ELT(x, i) (((SEXP *)(x)->data)[i])
#define SET_STRING_ELT(x, i, v) (((SEXP *)(x)->data)[i] = (v))
#define SET_VECTOR_ELT(x, i, v) (((SEXP *)(x)->data)[i] = (v))
#ifdef __cplusplus
}
#endif
#endif
