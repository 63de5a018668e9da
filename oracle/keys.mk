# oracle/keys.mk -- the reference side of the task keys (TEST INFRASTRUCTURE): _ref/libydref_keys.so is the reference
# harness (ref_harness.cc, as oracle/Makefile builds it) plus yd_derive_task_keys over flare's own Blake3 and EncodeHex
# and the vendored BLAKE3 C, all compiled verbatim from where they lie under $(REF) (ref_keys.cc).  Built only when
# $(REF) exists; reference sources are never copied into this repository.  BLAKE3 is built portable-only (no SIMD
# dispatch), which computes the same hash.
REF ?= /root/reference
CXX ?= g++
CC ?= gcc
CXXFLAGS ?= -std=gnu++2a -O2 -fPIC -Wall -Wno-sign-compare -Wno-unused-variable
INC = -I../include

REF_SRCS = $(REF)/yadcc/scheduler/task_dispatcher.cc \
           $(REF)/yadcc/scheduler/running_task_bookkeeper.cc \
           $(REF)/yadcc/common/parse_size.cc \
           $(REF)/flare/base/experimental/bloom_filter.cc \
           $(REF)/flare/base/crypto/blake3.cc \
           $(REF)/flare/base/encoding/hex.cc
REF_C_SRCS = $(REF)/thirdparty/xxhash/xxhash.c \
             $(REF)/thirdparty/blake3/blake3.c \
             $(REF)/thirdparty/blake3/blake3_dispatch.c \
             $(REF)/thirdparty/blake3/blake3_portable.c
BLAKE3_CFLAGS = -DBLAKE3_NO_SSE2 -DBLAKE3_NO_SSE41 -DBLAKE3_NO_AVX2 -DBLAKE3_NO_AVX512

all: ref_keys

ifneq ($(wildcard $(REF)/yadcc/scheduler/task_dispatcher.cc),)
ref_keys: _ref/libydref_keys.so
_ref/libydref_keys.so: ref_keys.cc ref_harness.cc $(wildcard ../include/*.h ../include/*.inc) $(REF_SRCS) \
                       $(wildcard shim/*/*.h shim/*/*/*.h shim/*/*/*/*.h shim_keys/*/*/*.h)
	mkdir -p _ref/keys
	for f in $(REF_C_SRCS); do $(CC) -O2 -fPIC $(BLAKE3_CFLAGS) -c -o _ref/keys/$$(basename $$f .c).o $$f || exit 1; done
	$(CXX) $(CXXFLAGS) -Ishim_keys -Ishim -I$(REF) -I$(REF)/thirdparty $(INC) -shared -o $@ ref_keys.cc $(REF_SRCS) \
	    $(foreach f,$(REF_C_SRCS),_ref/keys/$(basename $(notdir $(f))).o)
else
ref_keys:
	@echo "reference tree $(REF) not present: keeping prebuilt oracle/_ref/libydref_keys.so if any"
endif

.PHONY: all ref_keys
