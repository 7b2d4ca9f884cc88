# Host emulation with the calibrate_bridging_snvs kernels (test infrastructure; see emu_bsn.cpp).  g++ only.
#   make -f bridging_snvs.mk   -> _build/bsn/libugvc_emu_bsn.so   (what tests/test_bridging_snvs_emu_cpu.py loads)
# The other objects are the ones the main Makefile builds.
CSRC := ../../variantcalling_b200/csrc
B := _build/bsn
OUT := $(B)/libugvc_emu_bsn.so
CXXFLAGS := -O2 -std=c++17 -fPIC -pthread -w -Ishim_include -I$(CSRC)
BASE_OBJS := _build/emu_kernels.o _build/emu_capi.o _build/emu_multiallelic.o _build/hostio.o _build/collective.o

all: $(OUT)

base:
	$(MAKE) -f Makefile

$(BASE_OBJS): base

$(B)/emu_bsn.o: emu_bsn.cpp shim_include/cuda_runtime.h $(CSRC)/bridging_snvs.cu $(CSRC)/bridging_snvs.cuh $(CSRC)/low_af_ratio.cu $(CSRC)/low_af_ratio.cuh $(CSRC)/vcf_text.cuh $(CSRC)/numparse.h $(CSRC)/../../include/ugvc_b200.h
	@mkdir -p $(B)
	g++ $(CXXFLAGS) -x c++ -c emu_bsn.cpp -o $@

$(OUT): $(B)/emu_bsn.o $(BASE_OBJS)
	g++ -shared -O2 -o $@ $(B)/emu_bsn.o $(BASE_OBJS) -lz -lpthread -ldl

.PHONY: all base
