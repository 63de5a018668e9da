# Top-level build: the product library (CUDA, sm_90a only) and the CPU checkers.
#
#   make            -> yadcc_b200/libydsched.so + oracle/libydoracle.so (+ oracle/_ref if /root/reference exists)
#   make cuda       -> yadcc_b200/libydsched.so
#   make oracle     -> the checkers (+ checkers/libydport_state.so: the port with the state export / import)
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH = -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS = -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude -Iyadcc_b200/csrc
CSRC = yadcc_b200/csrc
LIB = yadcc_b200/libydsched.so

all: cuda oracle

cuda: $(LIB)

$(LIB): include/ydstate.h include/ydstate_codec.inc include/yddump_impl.inc $(CSRC)/ydsched.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.inc) include/ydshard.h include/ydsched.h include/ydsched_rpc_impl.inc include/ydservice.h include/ydservice_impl.inc include/ydwire.h include/ydwire_impl.inc
	$(NVCC) $(NVCCFLAGS) $(PTXAS_V) -shared -o $@ $(CSRC)/ydsched.cu -ldl

oracle: checkers/libydport_state.so
	$(MAKE) -C oracle all

checkers/libydport_state.so: checkers/port_state.cc oracle/port.cc include/ydstate.h include/ydstate_codec.inc include/ydsched.h $(wildcard include/*.inc)
	$(CXX) -std=gnu++2a -O2 -fPIC -Wall -Wno-sign-compare -Wno-unused-variable -Wno-subobject-linkage -Iinclude -shared -o $@ checkers/port_state.cc

clean:
	rm -f $(LIB) checkers/libydport_state.so
	$(MAKE) -C oracle clean

.PHONY: all cuda oracle clean
