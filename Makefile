# Builds everything in-tree: the product library (hand-written sm_90a (H100) CUDA behind the C ABI),
# the synthetic tipset builder and the CPU oracle (test infrastructure).
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
CSRC      := ipc_filecoin_proofs_b200/csrc
NVFLAGS   := -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr
CU_SRCS   := $(CSRC)/store.cu $(CSRC)/events.cu $(CSRC)/storage.cu $(CSRC)/storage_path.cu $(CSRC)/witness.cu $(CSRC)/prims.cu $(CSRC)/parallel.cu $(CSRC)/verify.cu $(CSRC)/json.cu $(CSRC)/json_parse.cu $(CSRC)/rpc_json.cu $(CSRC)/rpc_blocks.cu $(CSRC)/car.cu $(CSRC)/plan.cu $(CSRC)/resolve.cu $(CSRC)/actor.cu $(CSRC)/message_proof.cu $(CSRC)/capi.cu
CU_OBJS   := $(CU_SRCS:.cu=.o)
CU_HDRS   := $(wildcard $(CSRC)/*.cuh) include/ipcfp.h
LIB       := ipc_filecoin_proofs_b200/libipcfp.so

all: $(LIB) synth/libipcfp_synth.so oracle/liboracle.so

# objects depend on this file too: a change of NVFLAGS (the target architecture) rebuilds them
$(CSRC)/%.o: $(CSRC)/%.cu $(CU_HDRS) Makefile
	$(NVCC) $(NVFLAGS) $(EXTRA_NVFLAGS) -c $< -o $@

$(CSRC)/bundle_json.o: $(CSRC)/bundle_json.cpp include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -c $< -o $@

$(CSRC)/bundle_parse.o: $(CSRC)/bundle_parse.cpp $(CSRC)/json_value.h include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -c $< -o $@

$(CSRC)/rpc_parse.o: $(CSRC)/rpc_parse.cpp $(CSRC)/json_value.h include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -c $< -o $@

$(CSRC)/rpc_blocks_parse.o: $(CSRC)/rpc_blocks_parse.cpp $(CSRC)/json_value.h $(CSRC)/parsed_blocks.h include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -c $< -o $@

$(CSRC)/car_parse.o: $(CSRC)/car_parse.cpp $(CSRC)/parsed_blocks.h include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -c $< -o $@

# HIDE_INTERNALS=1 links with csrc/exports.map: only ipcfp_* stay in the dynamic symbol table (what a C-ABI library should export).
# Not the default yet: the default build is the one every GPU measurement and GPU test of round 2 ran on, and the change arrived after
# the round's GPU minutes were spent (tests/test_abi_layout.py checks the hidden build's export list and its C++-host behaviour on the CPU).
ifeq ($(HIDE_INTERNALS),1)
LIB_LDFLAGS := -Xlinker --version-script=$(CSRC)/exports.map
endif
LIB_OUT ?= $(LIB)

HOST_OBJS := $(CSRC)/bundle_json.o $(CSRC)/bundle_parse.o $(CSRC)/rpc_parse.o $(CSRC)/rpc_blocks_parse.o $(CSRC)/car_parse.o

$(LIB_OUT): $(CU_OBJS) $(HOST_OBJS) $(CSRC)/exports.map
	$(NVCC) -shared -gencode arch=compute_90a,code=sm_90a $(LIB_LDFLAGS) -o $@ $(CU_OBJS) $(HOST_OBJS) -lcudart -ldl

synth/libipcfp_synth.so: synth/synth.cpp synth/synth.h synth/cpu_crypto.h
	$(CXX) -O2 -std=c++17 -fPIC -shared -pthread -o $@ synth/synth.cpp

oracle/liboracle.so: oracle/oracle.cpp oracle/oracle.h synth/cpu_crypto.h include/ipcfp.h
	$(CXX) -O2 -std=c++17 -fPIC -shared -pthread -o $@ oracle/oracle.cpp

clean:
	rm -f $(CU_OBJS) $(HOST_OBJS) $(LIB) synth/libipcfp_synth.so oracle/liboracle.so

# The host-compiled device headers (tests/host_fuzz) and the JSON parser under AddressSanitizer + UBSan (DESIGN.md §7.12)
sanitize:
	IPCFP_HOST_FUZZ_SANITIZE=1 python -m pytest tests/test_host_fuzz.py tests/test_tail_bytes_host.py tests/test_bundle_json.py tests/test_json_items_host.py tests/test_json_unified_host.py tests/test_json_parse_host.py tests/test_rpc_json_host.py tests/test_rpc_blocks_host.py tests/test_car_host.py tests/test_plan_fetch_host.py tests/test_resolve_host.py tests/test_log_filter_host.py tests/test_log_bundle_host.py tests/test_message_proof_host.py tests/test_storage_paths_host.py tests/test_actor_host.py tests/test_message_proofs_host.py -q

.PHONY: all clean sanitize
