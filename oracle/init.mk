# oracle/init.mk -- builds the CPU oracle of include/cvb200_init.h (test infrastructure) into oracle/_build/, with oracle/Makefile's flags:
# -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_init.c composes
# ref_triangulation.c's triangulators and robustness test with ref_optimize.c's epipolar loss and three-view optimiser (which use
# ref_geom.c's eigen solver), so all of them are linked into this library.
#   make -C oracle -f init.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_init.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_init.so
$(OUT)/libcvb_oracle_init.so: $(SRCS) ref_triangulation.h ref_geom.h init.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_init.so
