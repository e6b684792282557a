# TEST INFRASTRUCTURE ONLY.  slopeavedown's checker, beside the others:
#   make -C oracle -f downslope.mk port   the C restatement oracle/port/libslopeavedown_oracle.so
#   make -C oracle -f downslope.mk ref    the reference's own slopeavedown, compiled UNCHANGED from /root/reference/src against the
#                                         MPI/GDAL shims into oracle/_ref/ next to the other reference tools
REF ?= /root/reference/src
OUT := _ref
CXX ?= g++
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -w -Ishim -I$(REF)

all: port ref
port: port/libslopeavedown_oracle.so
ref: $(OUT)/slopeavedown

port/libslopeavedown_oracle.so: port/slopeavedown_oracle.c
	gcc -O2 -fPIC -shared -ffp-contract=off -o $@ $< -lm
$(OUT)/shim.a:
	$(MAKE) -f Makefile $@
$(OUT)/slopeavedown: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/SlopeAveDownmn.cpp $(REF)/SlopeAveDown.cpp $(OUT)/shim.a -lz -lpthread -o $@
.PHONY: all port ref
