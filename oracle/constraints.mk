# oracle/constraints.mk -- builds the CPU oracle of include/cvb200_constraints.h (test infrastructure) into oracle/_build/, with
# oracle/Makefile's flags: -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).
# ref_constraints.c composes ref_triangulation.c's triangulators with ref_optimize.c's three-view optimiser (which use ref_geom.c's eigen
# solver), so all of them are linked into this library.  -fopenmp runs independent queries on several threads.
#   make -C oracle -f constraints.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_constraints.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_constraints.so
$(OUT)/libcvb_oracle_constraints.so: $(SRCS) ref_triangulation.h ref_geom.h constraints.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_constraints.so
