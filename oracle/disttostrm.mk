# TEST INFRASTRUCTURE ONLY.  d8hdisttostrm's and d8vdisttostrm's checker, beside the others:
#   make -C oracle -f disttostrm.mk port   the C restatement oracle/port/libdisttostrm_oracle.so
#   make -C oracle -f disttostrm.mk ref    the reference's own d8hdisttostrm and d8vdisttostrm, compiled UNCHANGED from
#                                          /root/reference/src against the MPI/GDAL shims into oracle/_ref/ next to the other tools
REF ?= /root/reference/src
OUT := _ref
CXX ?= g++
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -w -Ishim -I$(REF)

all: port ref
port: port/libdisttostrm_oracle.so
ref: $(OUT)/d8hdisttostrm $(OUT)/d8vdisttostrm

port/libdisttostrm_oracle.so: port/disttostrm_oracle.c
	gcc -O2 -fPIC -shared -ffp-contract=off -o $@ $< -lm
$(OUT)/shim.a:
	$(MAKE) -f Makefile $@
$(OUT)/d8hdisttostrm: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/D8HDistToStrmmn.cpp $(REF)/D8HDistToStrm.cpp $(OUT)/shim.a -lz -lpthread -o $@
$(OUT)/d8vdisttostrm: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/D8VDistToStrmmn.cpp $(REF)/D8VDistToStrm.cpp $(OUT)/shim.a -lz -lpthread -o $@
.PHONY: all port ref
