# Builds the CPU restatement of cgls! / crls! / lslq! (test infrastructure):  make -C oracle -f cgls.mk
# Same flags as the main oracle: -ffp-contract=off keeps every product rounded before its add (no implicit FMA).
CC = /usr/bin/gcc
CFLAGS = -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-function
all: libkrylov_oracle_cgls.so
libkrylov_oracle_cgls.so: krylov_oracle_cgls.c krylov_oracle_cgls.h krylov_oracle_lslq.h krylov_oracle_lsq.h krylov_oracle_impl.h
	$(CC) $(CFLAGS) -shared -o $@ krylov_oracle_cgls.c -lm
clean:
	rm -f libkrylov_oracle_cgls.so
