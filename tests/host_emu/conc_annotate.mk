# Host emulation with the concordance handle and its annotation kernel (test infrastructure; see emu_conc.cpp).  g++ only.
#   make -f conc_annotate.mk   -> _build/conc/libugvc_emu_conc.so   (what tests/test_conc_annotate_emu_cpu.py loads)
# The other kernel objects are the ones the main Makefile builds.
CSRC := ../../variantcalling_b200/csrc
B := _build/conc
OUT := $(B)/libugvc_emu_conc.so
CXXFLAGS := -O2 -std=c++17 -fPIC -pthread -w -Ishim_include -I$(CSRC)
BASE_OBJS := _build/emu_kernels.o _build/emu_multiallelic.o _build/hostio.o _build/collective.o

all: $(OUT)

base:
	$(MAKE) -f Makefile

$(BASE_OBJS): base

$(B)/emu_conc.o: emu_conc.cpp emu_capi.cpp shim_include/cuda_runtime.h $(CSRC)/capi.cu $(CSRC)/conc_handle.cu $(CSRC)/conc_annotate.cu $(CSRC)/concordance.cuh $(CSRC)/../../include/ugvc_b200.h
	@mkdir -p $(B)
	g++ $(CXXFLAGS) -x c++ -c emu_conc.cpp -o $@

$(OUT): $(B)/emu_conc.o $(BASE_OBJS)
	g++ -shared -O2 -o $@ $(B)/emu_conc.o $(BASE_OBJS) -lz -lpthread -ldl

.PHONY: all base
