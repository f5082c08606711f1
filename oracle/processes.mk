# Builds the CPU oracle of the Krylov processes (test infrastructure), with the flags of oracle/Makefile.  It links against
# the shared oracle library (built first by oracle/Makefile): the test knobs oracle_dot_mode / oracle_precond_block are
# that library's, so oracle.oracle.dot_mode switches these processes too.
CC = /usr/bin/gcc
CFLAGS = -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-function -fopenmp
all: libkrylov_oracle_processes.so
libkrylov_oracle_processes.so: krylov_oracle_processes.c krylov_oracle_processes.h krylov_oracle_impl.h libkrylov_oracle.so
	$(CC) $(CFLAGS) -shared -o $@ krylov_oracle_processes.c -L. -lkrylov_oracle -Wl,-rpath,'$$ORIGIN' -lm
clean:
	rm -f libkrylov_oracle_processes.so
