/* TEST INFRASTRUCTURE — minimal stand-in for R's <Rdefines.h> (see Rinternals.h here): the one macro the darknet
 * glue uses.  The test programs pass character vectors, so coercion is the identity. */
#ifndef ORACLE_STUB_RDEFINES_H
#define ORACLE_STUB_RDEFINES_H
#include "Rinternals.h"
#define AS_CHARACTER(x) (x)
#endif
