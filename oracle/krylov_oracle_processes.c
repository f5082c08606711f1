/*
 * krylov_oracle_processes.c -- TEST INFRASTRUCTURE ONLY.  The CPU restatement of the Krylov processes
 * (krylov_oracle_processes.h) on the shared BLAS-1 wrappers of krylov_oracle_impl.h, instantiated in Float64 and
 * Float32.  Built by oracle/processes.mk into oracle/libkrylov_oracle_processes.so, which links against the shared oracle
 * library and takes its test knobs (oracle_dot_mode, oracle_precond_block) from there: one dot_mode switch serves every
 * family.  Loaded by oracle/processes_oracle.py.  The product library (krylov.jl_b200/) never links, loads or calls this.
 */
#include <math.h>
#include <float.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

extern int oracle_precond_block;                 /* defined, with oracle_dot_mode, in libkrylov_oracle.so */

#define REAL double
#define SUF(name) name##_f64
#define SQRT sqrt
#define FABS fabs
#define COPYSIGN copysign
#define POW pow
#define EPS DBL_EPSILON
#define FLTMAX_OF DBL_MAX
#include "krylov_oracle_impl.h"
#include "krylov_oracle_processes.h"
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
#include "krylov_oracle_processes.h"
