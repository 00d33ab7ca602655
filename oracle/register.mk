# oracle/register.mk -- builds the CPU oracle of include/cvb200_register.h (test infrastructure) into oracle/_build/, with oracle/Makefile's
# flags: -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_register.c composes
# ref_match.c's exact k-NN, ref_geom.c's ARRSAC and P3P, ref_optimize.c's single-view optimiser and ref_triangulation.c's triangulators,
# so all of them are linked into this library.  Single-threaded (no -fopenmp: ref_match.c's pragma stays inert).
#   make -C oracle -f register.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_register.c ref_match.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_register.so
$(OUT)/libcvb_oracle_register.so: $(SRCS) ref_triangulation.h ref_geom.h ref_akaze.h register.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_register.so
