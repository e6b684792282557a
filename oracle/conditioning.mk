# TEST INFRASTRUCTURE ONLY.  flowdircond's and retlimflow's checkers, beside the others:
#   make -C oracle -f conditioning.mk port   the C restatements oracle/port/libconditioning_oracle.so
#   make -C oracle -f conditioning.mk ref    the reference's own flowdircond and retlimflow, compiled UNCHANGED from /root/reference/src against the
#                                            MPI/GDAL shims into oracle/_ref/ next to the other reference tools
REF ?= /root/reference/src
OUT := _ref
CXX ?= g++
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -w -Ishim -I$(REF)

all: port ref
port: port/libconditioning_oracle.so
ref: $(OUT)/flowdircond $(OUT)/retlimflow

port/libconditioning_oracle.so: port/conditioning_oracle.c
	gcc -O2 -fPIC -shared -ffp-contract=off -o $@ $< -lm
$(OUT)/shim.a:
	$(MAKE) -f Makefile $@
$(OUT)/flowdircond: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/flowdirconditionmn.cpp $(REF)/flowdircond.cpp $(OUT)/shim.a -lz -lpthread -o $@
$(OUT)/retlimflow: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/RetLimFlowmn.cpp $(REF)/RetlimFlow.cpp $(OUT)/shim.a -lz -lpthread -o $@
.PHONY: all port ref
