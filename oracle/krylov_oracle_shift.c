/*
 * krylov_oracle_shift.c -- TEST INFRASTRUCTURE ONLY.  The CPU restatement of the shift solvers
 * (krylov_oracle_shift.h: cg_lanczos_shift!, cgls_lanczos_shift!) on the helpers of krylov_oracle_impl.h, in Float64
 * and Float32: the one translation unit of libkrylov_oracle_shift.so (Makefile.shift), loaded by shift_oracle.py.
 * Its test knobs (dot mode, block-Jacobi M) are this library's own, set through shift_oracle.py.
 * The product library (krylov.jl_b200/) never links, loads or calls this.
 */
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

int oracle_dot_mode = 0;
void oracle_set_dot_mode(int m) { oracle_dot_mode = m; }
int oracle_precond_block = 0;
void oracle_set_precond_block(int bs) { oracle_precond_block = bs; }

#define REAL double
#define SUF(name) name##_f64
#define SQRT sqrt
#define FABS fabs
#define COPYSIGN copysign
#define POW pow
#define EPS DBL_EPSILON
#define FLTMAX_OF DBL_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_shift.h"
#undef REAL
#undef SUF
#undef SQRT
#undef FABS
#undef COPYSIGN
#undef POW
#undef EPS
#undef FLTMAX_OF

#define REAL float
#define SUF(name) name##_f32
#define SQRT sqrtf
#define FABS fabsf
#define COPYSIGN copysignf
#define POW powf
#define EPS FLT_EPSILON
#define FLTMAX_OF FLT_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_shift.h"
