# oracle/opt.mk -- builds the CPU oracle of include/cvb200_opt.h (test infrastructure) into oracle/_build/, with oracle/Makefile's flags:
# -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).  ref_optimize_l1.c uses
# ref_optimize.c's gradients (which use ref_geom.c's triangulation), so both are linked into this library as well.
#   make -C oracle -f opt.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -fopenmp -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_optimize_l1.c ref_optimize.c ref_geom.c
all: $(OUT)/libcvb_oracle_opt.so
$(OUT)/libcvb_oracle_opt.so: $(SRCS) ref_optimize_l1.h ref_geom.h opt.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_opt.so
