# oracle/image.mk -- builds the CPU oracle of include/cvb200_image.h (test infrastructure) into oracle/_build/, with oracle/Makefile's
# flags (-fno-fast-math: the division by 255 / 65535 is the correctly rounded one).
#   make -C oracle -f image.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -ffp-contract=off -fno-fast-math -Wall
OUT = _build
all: $(OUT)/libcvb_oracle_image.so
$(OUT)/libcvb_oracle_image.so: ref_image.c ref_image.h image.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ ref_image.c
clean:
	rm -f $(OUT)/libcvb_oracle_image.so
