# Builds the CPU oracle of cgne! and crmr! (test infrastructure), with the flags of oracle/Makefile.  It links against
# the shared oracle library (built first by oracle/Makefile): the test knobs oracle_dot_mode / oracle_precond_block are
# that library's, so oracle.oracle.dot_mode switches these solvers too.
CC = /usr/bin/gcc
CFLAGS = -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-function -fopenmp
all: libkrylov_oracle_cgne.so
libkrylov_oracle_cgne.so: krylov_oracle_cgne.c krylov_oracle_cgne.h krylov_oracle_impl.h libkrylov_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ krylov_oracle_cgne.c -L. -lkrylov_oracle -Wl,-rpath,'$$ORIGIN' -lm
clean:
	rm -f libkrylov_oracle_cgne.so
