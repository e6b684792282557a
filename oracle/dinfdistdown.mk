# TEST INFRASTRUCTURE ONLY.  dinfdistdown's checker, beside the others:
#   make -C oracle -f dinfdistdown.mk port   the C restatement oracle/port/libdinfdistdown_oracle.so
#   make -C oracle -f dinfdistdown.mk ref    the reference's own dinfdistdown, compiled UNCHANGED from /root/reference/src against
#                                            the MPI/GDAL shims (commonLib.cpp, which provides prop(), comes with the shim library)
#                                            into oracle/_ref/ next to the other tools
REF ?= /root/reference/src
OUT := _ref
CXX ?= g++
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -w -Ishim -I$(REF)

all: port ref
port: port/libdinfdistdown_oracle.so
ref: $(OUT)/dinfdistdown

port/libdinfdistdown_oracle.so: port/dinfdistdown_oracle.c
	gcc -O2 -fPIC -shared -ffp-contract=off -o $@ $< -lm
$(OUT)/shim.a:
	$(MAKE) -f Makefile $@
$(OUT)/dinfdistdown: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/DinfDistDownmn.cpp $(REF)/DinfDistDown.cpp $(OUT)/shim.a -lz -lpthread -o $@
.PHONY: all port ref
