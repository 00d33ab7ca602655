# oracle/incorporate.mk -- builds the CPU oracle of include/cvb200_incorporate.h's two CSR edits (test infrastructure) into oracle/_build/,
# with oracle/Makefile's flags.  ref_incorporate.c stands alone: the chain's other stages are the register, constraints and
# reconstruction oracles, composed in oracle/pyoracle_incorporate.py.
#   make -C oracle -f incorporate.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_incorporate.c
all: $(OUT)/libcvb_oracle_incorporate.so
$(OUT)/libcvb_oracle_incorporate.so: $(SRCS) incorporate.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_incorporate.so
