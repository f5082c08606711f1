# Builds the CPU restatement of bilq! / qmr! (test infrastructure):  make -C oracle -f biorth.mk
# Same flags as the main oracle: -ffp-contract=off keeps every product rounded before its add (no implicit FMA).
CC = /usr/bin/gcc
CFLAGS = -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-function
all: libkrylov_oracle_biorth.so
libkrylov_oracle_biorth.so: krylov_oracle_biorth.c krylov_oracle_biorth.h krylov_oracle_impl.h
	$(CC) $(CFLAGS) -shared -o $@ krylov_oracle_biorth.c -lm
clean:
	rm -f libkrylov_oracle_biorth.so
