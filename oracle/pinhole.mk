# oracle/pinhole.mk -- builds the CPU oracle of include/cvb200_pinhole.h (test infrastructure) into oracle/_build/, with oracle/Makefile's
# flags: -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_pinhole.c uses
# the relative triangulators of ref_triangulation.c and the essential routines of ref_geom.c, so both (and ref_optimize.c, which
# ref_triangulation.c needs) are linked into this library as well.
#   make -C oracle -f pinhole.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_pinhole.c ref_triangulation.c ref_geom.c ref_optimize.c
all: $(OUT)/libcvb_oracle_pinhole.so
$(OUT)/libcvb_oracle_pinhole.so: $(SRCS) ref_pinhole.h ref_triangulation.h ref_geom.h pinhole.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_pinhole.so
