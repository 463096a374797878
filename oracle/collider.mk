# Builds the CPU oracle with the signed-distance collider (test infrastructure only; never linked by the product).
# Same compiler and flags as the oracle's Makefile: collider_oracle.c compiles claymore_oracle.c into its own translation unit.
CC := $(shell test -x /usr/bin/gcc && echo /usr/bin/gcc || echo gcc)
CFLAGS ?= -O2 -std=c99 -fPIC -fopenmp -ffp-contract=off -fno-fast-math -Wall -Wextra -Wno-unused-parameter
all: libclaymore_collider_oracle.so
libclaymore_collider_oracle.so: collider_oracle.c collider_oracle.h claymore_oracle.c claymore_oracle.h
	$(CC) $(CFLAGS) -shared -o $@ collider_oracle.c -lm
clean:
	rm -f libclaymore_collider_oracle.so
