# Host emulation with the filter_low_af_ratio_to_background kernels (test infrastructure; see emu_afr.cpp).  g++ only.
#   make -f low_af_ratio.mk   -> _build/afr/libugvc_emu_afr.so   (what tests/test_low_af_ratio_emu_cpu.py loads)
# The other objects are the ones the main Makefile builds.
CSRC := ../../variantcalling_b200/csrc
B := _build/afr
OUT := $(B)/libugvc_emu_afr.so
CXXFLAGS := -O2 -std=c++17 -fPIC -pthread -w -Ishim_include -I$(CSRC)
BASE_OBJS := _build/emu_kernels.o _build/emu_capi.o _build/emu_multiallelic.o _build/hostio.o _build/collective.o

all: $(OUT)

base:
	$(MAKE) -f Makefile

$(BASE_OBJS): base

$(B)/emu_afr.o: emu_afr.cpp shim_include/cuda_runtime.h $(CSRC)/low_af_ratio.cu $(CSRC)/low_af_ratio.cuh $(CSRC)/numparse.h $(CSRC)/../../include/ugvc_b200.h
	@mkdir -p $(B)
	g++ $(CXXFLAGS) -x c++ -c emu_afr.cpp -o $@

$(OUT): $(B)/emu_afr.o $(BASE_OBJS)
	g++ -shared -O2 -o $@ $(B)/emu_afr.o $(BASE_OBJS) -lz -lpthread -ldl

.PHONY: all base
