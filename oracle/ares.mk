# Builds the CPU restatement of car! / minares! (test infrastructure):  make -C oracle -f ares.mk
# Same flags as the main oracle: -ffp-contract=off keeps every product rounded before its add (no implicit FMA).
CC = /usr/bin/gcc
CFLAGS = -O2 -fPIC -std=c11 -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-function
all: libkrylov_oracle_ares.so
libkrylov_oracle_ares.so: krylov_oracle_ares.c krylov_oracle_ares.h krylov_oracle_impl.h
	$(CC) $(CFLAGS) -shared -o $@ krylov_oracle_ares.c -lm
clean:
	rm -f libkrylov_oracle_ares.so
