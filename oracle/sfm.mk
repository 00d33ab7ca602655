# oracle/sfm.mk -- builds the CPU oracle of include/cvb200_sfm.h (test infrastructure) into oracle/_build/, with oracle/Makefile's flags:
# -ffp-contract=off: no fused multiply-add anywhere (matches a default x86-64 Rust build of the reference).
#   make -C oracle -f sfm.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall
OUT = _build
all: $(OUT)/libcvb_oracle_sfm.so
$(OUT)/libcvb_oracle_sfm.so: ref_sfm.c sfm.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ ref_sfm.c -lm
clean:
	rm -f $(OUT)/libcvb_oracle_sfm.so
