# Top-level build: the product library (CUDA, sm_90a only) and the CPU checkers.
#
#   make            -> yadcc_b200/libydsched.so + oracle/libydoracle.so (+ oracle/_ref if /root/reference exists)
#   make cuda       -> yadcc_b200/libydsched.so
#   make oracle     -> the checkers (+ checkers/libydport_state.so: the port with the state export / import,
#                      checkers/libydport_keys.so and oracle/_ref/libydref_keys.so: port and reference with the task keys)
#   make fake_nccl  -> tests/fake_nccl/libnccl.so.2: the test-only NCCL stand-in that runs several ranks of the
#                      range-sharded scheduler as threads of one process on one GPU (tests/test_shard_one_gpu.py)
#   make primitives -> tests/kernels/libydprim.so: host wrappers that launch the product's device primitives on their own
#                      (tests/test_device_primitives.py)
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH = -gencode arch=compute_90a,code=sm_90a
NVCCFLAGS = -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-unused-function -Iinclude -Iyadcc_b200/csrc
CSRC = yadcc_b200/csrc
LIB = yadcc_b200/libydsched.so

all: cuda oracle fake_nccl primitives

cuda: $(LIB)

$(LIB): include/ydstate.h include/ydkeys.h include/ydstate_codec.inc include/yddump_impl.inc include/ydsched_keys_impl.inc $(CSRC)/ydsched.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.inc) include/ydshard.h include/ydfilter_packed.h include/ydrpcs_packed.h include/ydruns.h include/ydsched.h include/ydsched_rpc_impl.inc include/ydservice.h include/ydservice_impl.inc include/ydwire.h include/ydwire_impl.inc
	$(NVCC) $(NVCCFLAGS) $(PTXAS_V) -shared -o $@ $(CSRC)/ydsched.cu -ldl

oracle: checkers/libydport_state.so checkers/libydport_keys.so
	$(MAKE) -C oracle all
	$(MAKE) -C oracle -f keys.mk all

checkers/libydport_state.so: checkers/port_state.cc oracle/port.cc include/ydstate.h include/ydstate_codec.inc include/ydsched.h include/ydfilter_packed.h include/ydrpcs_packed.h include/ydruns.h $(wildcard include/*.inc)
	$(CXX) -std=gnu++2a -O2 -fPIC -Wall -Wno-sign-compare -Wno-unused-variable -Wno-subobject-linkage -Iinclude -shared -o $@ checkers/port_state.cc

checkers/libydport_keys.so: checkers/port_keys.cc oracle/port.cc include/ydsched.h include/ydkeys.h include/ydfilter_packed.h include/ydrpcs_packed.h include/ydruns.h $(wildcard include/*.inc)
	$(CXX) -std=gnu++2a -O2 -fPIC -Wall -Wno-sign-compare -Wno-unused-variable -Wno-subobject-linkage -Iinclude -shared -o $@ checkers/port_keys.cc

FAKE_NCCL = tests/fake_nccl/libnccl.so.2
fake_nccl: $(FAKE_NCCL)

$(FAKE_NCCL): tests/fake_nccl/fake_nccl.cc
	$(CXX) -std=c++17 -O2 -fPIC -Wall -shared -Wl,-soname,libnccl.so.2 -o $@ $< -ldl -pthread

PRIM = tests/kernels/libydprim.so
primitives: $(PRIM)

$(PRIM): tests/kernels/primitives.cu $(CSRC)/radix.cuh $(CSRC)/filter.cuh $(CSRC)/state.cuh $(CSRC)/common.cuh include/ydsched.h include/ydstate.h
	$(NVCC) $(NVCCFLAGS) -shared -o $@ tests/kernels/primitives.cu

clean:
	rm -f $(LIB) $(FAKE_NCCL) $(PRIM) checkers/libydport_state.so checkers/libydport_keys.so oracle/_ref/libydref_keys.so
	$(MAKE) -C oracle clean

.PHONY: all cuda oracle fake_nccl primitives clean
