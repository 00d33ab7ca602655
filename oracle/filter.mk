# oracle/filter.mk -- builds the CPU oracle of include/cvb200_filter.h's filters (test infrastructure) into oracle/_build/, with
# oracle/Makefile's flags (-ffp-contract=off: every multiply and add rounds on its own, as the reference's f32x4 lanes do).
#   make -C oracle -f filter.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall
OUT = _build
all: $(OUT)/libcvb_oracle_filter.so
$(OUT)/libcvb_oracle_filter.so: ref_filter.c filter.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ ref_filter.c
clean:
	rm -f $(OUT)/libcvb_oracle_filter.so
