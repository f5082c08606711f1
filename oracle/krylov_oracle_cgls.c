/*
 * krylov_oracle_cgls.c -- TEST INFRASTRUCTURE ONLY.  CPU restatement of cgls!, crls! (krylov_oracle_cgls.h) and lslq!
 * (krylov_oracle_lslq.h) on the
 * BLAS-1 wrappers and to_boundary of krylov_oracle_impl.h and the rectangular products of krylov_oracle_lsq.h, built as
 * its own library (oracle/cgls.mk -> oracle/libkrylov_oracle_cgls.so) and loaded by oracle/cgls_oracle.py.
 * The product library (krylov.jl_b200/) never links, loads or calls this.
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* knobs of krylov_oracle_impl.h, fixed at their defaults here (sequential sums, diagonal preconditioners) */
int oracle_dot_mode = 0;
int oracle_precond_block = 0;

/* ---- Float64 instantiation ---- */
#define REAL double
#define SUF(name) name##_f64
#define SQRT sqrt
#define FABS fabs
#define COPYSIGN copysign
#define POW pow
#define EPS DBL_EPSILON
#define FLTMAX_OF DBL_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_lsq.h"
#include "krylov_oracle_cgls.h"
#include "krylov_oracle_lslq.h"
#undef REAL
#undef SUF
#undef SQRT
#undef FABS
#undef COPYSIGN
#undef POW
#undef EPS
#undef FLTMAX_OF

/* ---- Float32 instantiation ---- */
#define REAL float
#define SUF(name) name##_f32
#define SQRT sqrtf
#define FABS fabsf
#define COPYSIGN copysignf
#define POW powf
#define EPS FLT_EPSILON
#define FLTMAX_OF FLT_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_lsq.h"
#include "krylov_oracle_cgls.h"
#include "krylov_oracle_lslq.h"
