# oracle/export.mk -- builds the CPU oracle of include/cvb200_export.h (test infrastructure) into oracle/_build/, with oracle/Makefile's
# flags: -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_export.c composes
# ref_triangulation.c's triangulators (which use ref_geom.c's eigen solver and ref_optimize.c), so all of them are linked into this
# library.  -fopenmp runs the landmarks, and the views, on several threads.
#   make -C oracle -f export.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_export.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_export.so
$(OUT)/libcvb_oracle_export.so: $(SRCS) ref_triangulation.h ref_geom.h export.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_export.so
