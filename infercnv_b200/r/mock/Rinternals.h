/* Minimal mock of R's C API - ONLY so tests/test_r_shim_compiles.py can type-check
 * infercnvb200_shim.c in an image without R.  Never linked into anything. */
#ifndef MOCK_RINTERNALS_H
#define MOCK_RINTERNALS_H
#include <stddef.h>
typedef struct SEXPREC *SEXP;
typedef void *(*DL_FUNC)(void);
typedef struct _DllInfo DllInfo;
typedef ptrdiff_t R_xlen_t;
typedef struct { const char *name; DL_FUNC fun; int numArgs; } R_CallMethodDef;
#define LGLSXP 10
#define REALSXP 14
#define INTSXP 13
#define VECSXP 19
#define FALSE 0
extern SEXP R_DimSymbol;
extern SEXP R_NilValue;
SEXP Rf_getAttrib(SEXP, SEXP);
int *INTEGER(SEXP);
int *LOGICAL(SEXP);
double *REAL(SEXP);
int Rf_length(SEXP);
R_xlen_t Rf_xlength(SEXP);
SEXP VECTOR_ELT(SEXP, long);
SEXP SET_VECTOR_ELT(SEXP, long, SEXP);
SEXP Rf_allocMatrix(unsigned, int, int);
SEXP Rf_allocVector(unsigned, long);
SEXP Rf_protect(SEXP);
void Rf_unprotect(int);
#define PROTECT(s) Rf_protect(s)
#define UNPROTECT(n) Rf_unprotect(n)
int Rf_asLogical(SEXP);
int Rf_asInteger(SEXP);
double Rf_asReal(SEXP);
int Rf_isNull(SEXP);
SEXP Rf_ScalarLogical(int);
SEXP Rf_ScalarInteger(int);
void Rf_error(const char *, ...) __attribute__((noreturn));
int R_registerRoutines(DllInfo *, const void *, const R_CallMethodDef *, const void *, const void *);
int R_useDynamicSymbols(DllInfo *, int);
#endif
