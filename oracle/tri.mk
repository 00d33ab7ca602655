# oracle/tri.mk -- builds the CPU oracle of include/cvb200_tri.h (test infrastructure) into oracle/_build/, with oracle/Makefile's flags:
# -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_triangulation.c uses
# ref_geom.c's symmetric eigen solver and ref_optimize.c's epipolar loss, so both are linked into this library as well.
#   make -C oracle -f tri.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_tri.so
$(OUT)/libcvb_oracle_tri.so: $(SRCS) ref_triangulation.h ref_geom.h tri.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_tri.so
