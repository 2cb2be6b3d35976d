# oracle/read_provider.mk -- the reference's read input as a test oracle (nothing here is shipped).
#
#   _ref/libngmlr_reads.so   oracle/read_provider_shim.cpp linked against _ref/libngmlr_full.so (built by
#                            oracle/Makefile's `ref` target, whose objects are the UNMODIFIED reference sources).
# Only built where $(REF) exists, like the other reference oracles.
REF ?= /root/reference
SSW := $(REF)/lib/Complete-Striped-Smith-Waterman-Library/src

all:
	@if [ -d $(REF)/src ]; then $(MAKE) -f read_provider.mk _ref/libngmlr_reads.so; else echo "reference not present; skipping oracle/_ref/libngmlr_reads.so"; fi

_ref/libngmlr_reads.so: read_provider_shim.cpp _ref/libngmlr_full.so
	g++ -O2 -g -DNDEBUG -std=c++11 -fPIC -w -shared -I$(REF)/src -I$(REF)/lib -I$(SSW) -o $@ read_provider_shim.cpp \
	    -L_ref -l:libngmlr_full.so -Wl,-rpath,'$$ORIGIN' -lz -lpthread
