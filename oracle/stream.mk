# TEST INFRASTRUCTURE ONLY.  The reference's two stream-definition tools, peukerdouglas and lengtharea, compiled UNCHANGED from
# /root/reference/src against the MPI/GDAL shims into oracle/_ref/ next to the others (make -C oracle ref builds the shims first):
#   make -C oracle -f stream.mk
REF ?= /root/reference/src
OUT := _ref
CXX ?= g++
CXXFLAGS := -std=c++17 -O3 -DNDEBUG -w -Ishim -I$(REF)

all: $(OUT)/peukerdouglas $(OUT)/lengtharea

$(OUT)/shim.a:
	$(MAKE) -f Makefile $@
$(OUT)/peukerdouglas: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/PeukerDouglasmn.cpp $(REF)/PeukerDouglas.cpp $(OUT)/shim.a -lz -lpthread -o $@
$(OUT)/lengtharea: $(OUT)/shim.a
	$(CXX) $(CXXFLAGS) $(REF)/LengthAreamn.cpp $(REF)/LengthArea.cpp $(OUT)/shim.a -lz -lpthread -o $@
.PHONY: all
