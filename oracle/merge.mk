# oracle/merge.mk -- builds the CPU oracle of include/cvb200_merge.h's move edit (test infrastructure) into oracle/_build/, with
# oracle/Makefile's flags.  ref_merge.c stands alone: the merge's other stages are the register, incorporate, constraints and
# reconstruction oracles, composed in oracle/pyoracle_merge.py.
#   make -C oracle -f merge.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_merge.c
all: $(OUT)/libcvb_oracle_merge.so
$(OUT)/libcvb_oracle_merge.so: $(SRCS) merge.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_merge.so
