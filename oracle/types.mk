# oracle/types.mk -- builds the CLancIR element-type oracles (TEST INFRASTRUCTURE, not product):
#
#   _ref/liblancir_types_ref.so   upstream lancir.h compiled from REF through lancir_types_shim.cpp with the
#                                 pinned flags.  Only built when REF exists (the prebuilt .so travels with
#                                 the tree elsewhere).
#   liblancir_types_port.so       avir_port.c's CLancIR with every element type's load and output stage
#                                 (lancir_types_port.c).

REF ?= /root/reference
CXX ?= g++
CC ?= gcc
PIN = -O2 -mavx2 -ffp-contract=off

all: port ref

port: liblancir_types_port.so

liblancir_types_port.so: lancir_types_port.c avir_port.c
	$(CC) -std=c11 -O2 -ffp-contract=off -fPIC -shared -o $@ lancir_types_port.c avir_port.c -lm

ref:
	@if [ -f $(REF)/lancir.h ]; then $(MAKE) -f types.mk _ref/liblancir_types_ref.so; \
	else echo "oracle: $(REF) absent -- using prebuilt oracle/_ref"; fi

_ref/liblancir_types_ref.so: lancir_types_shim.cpp
	mkdir -p _ref
	$(CXX) -std=c++17 $(PIN) -fPIC -shared -I$(REF) -o $@ $<

clean:
	rm -f _ref/liblancir_types_ref.so liblancir_types_port.so

.PHONY: all port ref clean
