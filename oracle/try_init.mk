# oracle/try_init.mk -- builds the CPU oracle of include/cvb200_try_init.h's add_reconstruction (test infrastructure) into oracle/_build/,
# with oracle/Makefile's flags.  ref_try_init.c stands alone: try_init's other stage is the init oracle, composed in
# oracle/pyoracle_try_init.py.
#   make -C oracle -f try_init.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall -Wno-unknown-pragmas
OUT = _build
SRCS = ref_try_init.c
all: $(OUT)/libcvb_oracle_try_init.so
$(OUT)/libcvb_oracle_try_init.so: $(SRCS) try_init.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ $(SRCS) -lm
clean:
	rm -f $(OUT)/libcvb_oracle_try_init.so
