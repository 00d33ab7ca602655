# oracle/stages.mk -- builds the CPU oracle of include/cvb200_stages.h's describe call (test infrastructure) into oracle/_build/, with
# oracle/Makefile's floating-point flags (no contraction: the reference's unfused f32 arithmetic; REF_LIBM_FMA selects glibc's FMA
# sinf / cosf variant through explicit fma() calls).
#   make -C oracle -f stages.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall
OUT = _build
all: $(OUT)/libcvb_oracle_stages.so
$(OUT)/libcvb_oracle_stages.so: ref_stages.c ref_akaze.h ref_libm.h stages.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ ref_stages.c -lm
clean:
	rm -f $(OUT)/libcvb_oracle_stages.so
