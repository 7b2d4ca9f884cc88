# Host emulation with the gvcf_hcr kernels (test infrastructure; see emu_hcr.cpp).  g++ only.
#   make -f gvcf_hcr.mk   -> _build/hcr/libugvc_emu_hcr.so   (what tests/test_gvcf_hcr_emu_cpu.py loads)
# The other objects are the ones the main Makefile builds.
CSRC := ../../variantcalling_b200/csrc
B := _build/hcr
OUT := $(B)/libugvc_emu_hcr.so
CXXFLAGS := -O2 -std=c++17 -fPIC -pthread -w -Ishim_include -I$(CSRC)
BASE_OBJS := _build/emu_kernels.o _build/emu_capi.o _build/emu_multiallelic.o _build/hostio.o _build/collective.o

all: $(OUT)

base:
	$(MAKE) -f Makefile

$(BASE_OBJS): base

$(B)/emu_hcr.o: emu_hcr.cpp shim_include/cuda_runtime.h $(CSRC)/gvcf_hcr.cu $(CSRC)/gvcf_hcr.cuh $(CSRC)/low_af_ratio.cu $(CSRC)/low_af_ratio.cuh $(CSRC)/vcf_text.cuh $(CSRC)/numparse.h $(CSRC)/../../include/ugvc_b200.h
	@mkdir -p $(B)
	g++ $(CXXFLAGS) -x c++ -c emu_hcr.cpp -o $@

$(OUT): $(B)/emu_hcr.o $(BASE_OBJS)
	g++ -shared -O2 -o $@ $(B)/emu_hcr.o $(BASE_OBJS) -lz -lpthread -ldl

.PHONY: all base
