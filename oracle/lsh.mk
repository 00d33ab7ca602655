# oracle/lsh.mk -- builds the CPU oracle of include/cvb200_lsh.h's similar-frame search (test infrastructure) into oracle/_build/, with
# oracle/Makefile's flags (-fopenmp: one query per thread, as oracle/ref_match.c does).
#   make -C oracle -f lsh.mk
CC = gcc
CFLAGS = -O3 -march=x86-64-v3 -fPIC -fopenmp -Wall
OUT = _build
all: $(OUT)/libcvb_oracle_lsh.so
$(OUT)/libcvb_oracle_lsh.so: ref_lsh.c lsh.mk
	mkdir -p $(OUT)
	$(CC) $(CFLAGS) -shared -o $@ ref_lsh.c
clean:
	rm -f $(OUT)/libcvb_oracle_lsh.so
