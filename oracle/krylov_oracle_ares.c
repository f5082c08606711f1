/*
 * krylov_oracle_ares.c -- TEST INFRASTRUCTURE ONLY.  CPU restatement of car! and minares! (krylov_oracle_ares.h) on
 * the BLAS-1 wrappers of krylov_oracle_impl.h, built as its own library (oracle/ares.mk ->
 * oracle/libkrylov_oracle_ares.so) and loaded by oracle/ares_oracle.py.
 * The product library (krylov.jl_b200/) never links, loads or calls this.
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* knobs of krylov_oracle_impl.h: the dot-product mode is settable (Float32 envelope tests); diagonal preconditioners */
int oracle_dot_mode = 0;
void oracle_set_dot_mode(int m) { oracle_dot_mode = m; }
int oracle_precond_block = 0;

/* ---- Float64 instantiation ---- */
#define REAL double
#define SUF(name) name##_f64
#define SQRT sqrt
#define FABS fabs
#define COPYSIGN copysign
#define POW pow
#define EPS DBL_EPSILON
#include "krylov_oracle_impl.h"
#include "krylov_oracle_ares.h"
#undef REAL
#undef SUF
#undef SQRT
#undef FABS
#undef COPYSIGN
#undef POW
#undef EPS

/* ---- Float32 instantiation ---- */
#define REAL float
#define SUF(name) name##_f32
#define SQRT sqrtf
#define FABS fabsf
#define COPYSIGN copysignf
#define POW powf
#define EPS FLT_EPSILON
#include "krylov_oracle_impl.h"
#include "krylov_oracle_ares.h"
