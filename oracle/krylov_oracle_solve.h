/*
 * krylov_oracle_solve.h -- TEST INFRASTRUCTURE ONLY (same status as krylov_oracle_impl.h; include it after every
 * solver family's header, instantiated by krylov_oracle.c).  The one exported solve entry: the table from a solver's
 * Krylov.jl name to its body, and, for the bodies two solvers share, which of the two it runs (variant).
 */
typedef int (*SUF(solver_body))(int variant, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out,
                                oracle_stats *st);

static const struct {
  const char *name;
  SUF(solver_body) body;
  int variant;
} SUF(solvers)[] = {
  {"cg", SUF(cg), 0},           {"bicgstab", SUF(bicgstab), 0}, {"gmres", SUF(gmres), 0},
  {"minres", SUF(minres), 0},   {"cgs", SUF(cgs), 0},           {"cg_lanczos", SUF(cg_lanczos), 0},
  {"fom", SUF(fom), 0},         {"fgmres", SUF(fgmres), 0},     {"dqgmres", SUF(dqgmres), 0},
  {"diom", SUF(diom), 0},       {"cr", SUF(cr), 0},             {"car", SUF(car), 0},
  {"minares", SUF(minares), 0}, {"bilq", SUF(biorth), 0},       {"qmr", SUF(biorth), 1},
  {"bilqr", SUF(adjoint), 0},   {"trilqr", SUF(adjoint), 1},    {"lsqr", SUF(lsq), 0},
  {"lsmr", SUF(lsq), 1},        {"cgls", SUF(cgls), 0},         {"crls", SUF(cgls), 1},
  {"lslq", SUF(lslq), 0},       {"craig", SUF(leastnorm), 0},   {"craigmr", SUF(leastnorm), 1},
  {"lnlq", SUF(lnlq), 0},       {"cgne", SUF(cgne), 0},         {"crmr", SUF(crmr), 0},
};

/* Runs solver `name` on P with options o into out and st.  Returns the body's code (0, or where the reference
 * raises: the family's error code), or -1 for a name not in the table. */
int SUF(oracle_solve)(const char *name, const SUF(problem) *P, const oracle_options *o, SUF(outputs) *out,
                      oracle_stats *st) {
  for (size_t i = 0; i < sizeof(SUF(solvers)) / sizeof(SUF(solvers)[0]); i++)
    if (!strcmp(name, SUF(solvers)[i].name)) return SUF(solvers)[i].body(SUF(solvers)[i].variant, P, o, out, st);
  return -1;
}
