# oracle/reconstruction.mk -- builds the CPU oracle of include/cvb200_reconstruction.h (test infrastructure) into oracle/_build/, with
# oracle/Makefile's flags: -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).
# ref_reconstruction.c composes ref_triangulation.c's triangulators (which use ref_geom.c's eigen solver) with ref_optimize.c's epipolar
# loss, so all of them are linked into this library.  -fopenmp runs the views of a step and the landmarks of a filter on several threads.
#   make -C oracle -f reconstruction.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_reconstruction.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_reconstruction.so
$(OUT)/libcvb_oracle_reconstruction.so: $(SRCS) ref_triangulation.h ref_geom.h reconstruction.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_reconstruction.so
