# Builds the product library (CUDA, sm_90a) and the CPU oracle (test infrastructure).
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
CC        ?= gcc
PKG       := clarabel.rs_b200
CSRC      := $(PKG)/csrc
LIB       := $(PKG)/libclarabel_b200.so
ORACLE    := oracle/liboracle.so
GENCODE   := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -O3 -std=c++17 -lineinfo --extended-lambda $(GENCODE) -Xcompiler -fPIC,-O3,-Wall -Xptxas -v
CU_SRCS   := $(wildcard $(CSRC)/*.cu)
CPP_SRCS  := $(wildcard $(CSRC)/*.cpp)
CU_OBJS   := $(CU_SRCS:.cu=.o)
CPP_OBJS  := $(CPP_SRCS:.cpp=.o)
HDRS      := $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.cuh) include/clarabel_b200.h
ORACLE_SRCS := $(wildcard oracle/*.c)

all: $(LIB) $(ORACLE)

$(CSRC)/%.o: $(CSRC)/%.cu $(HDRS)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(CSRC)/%.o: $(CSRC)/%.cpp $(HDRS)
	$(CXX) -O3 -std=c++17 -fPIC -Wall -pthread -c $< -o $@

$(LIB): $(CU_OBJS) $(CPP_OBJS)
	$(NVCC) -shared $(GENCODE) -o $@ $^ -lcudart -lpthread -ldl

$(ORACLE): $(ORACLE_SRCS) $(wildcard oracle/*.h)
	$(CC) -O3 -march=x86-64-v3 -fPIC -shared -Wall -o $@ $(ORACLE_SRCS) -lm

clean:
	rm -f $(CSRC)/*.o $(LIB) $(ORACLE) tests/host_harness/*.so

.PHONY: all clean

# host build of the nonsymmetric cones' thread bodies (test infrastructure, see tests/host_harness/ns3_host.cpp)
HARNESS := tests/host_harness/libns3_host.so
$(HARNESS): tests/host_harness/ns3_host.cpp $(CSRC)/cones_nonsym.cuh
	$(CXX) -O2 -std=c++17 -fPIC -shared -Wall -o $@ $<
all: $(HARNESS)

# CUDA-runtime stand-in for LD_PRELOAD in a test subprocess (host-side setup checks without a GPU, see the file header)
FAKERT := tests/host_harness/libfake_cudart.so
$(FAKERT): tests/host_harness/fake_cudart.c
	$(CC) -O1 -fPIC -shared -Wall -o $@ $<
all: $(FAKERT)

# CUDA-on-CPU emulated builds (test infrastructure, see tests/emu/cuda_emu.h): the .cu sources AND the csrc headers are
# rewritten into tests/emu/gen/ (launch syntax, __shared__ storage); libclarabel_emu.so has a dense host LDL behind
# the LDLObject interface, libclarabel_emu_full.so runs the multifrontal kernels of ldl.cu too.
EMU      := tests/emu/libclarabel_emu.so
EMU_FULL := tests/emu/libclarabel_emu_full.so
EMU_HDRS := $(patsubst $(CSRC)/%,tests/emu/gen/%,$(wildcard $(CSRC)/*.h $(CSRC)/*.cuh))
EMU_GEN  := tests/emu/gen/cones.cpp tests/emu/gen/cones_psd.cpp tests/emu/gen/cones_nonsym.cpp tests/emu/gen/solver.cpp
EMU_FLAGS := -O1 -g -march=x86-64-v3 -ffp-contract=fast -std=c++17 -fPIC -shared -pthread -Wno-unknown-pragmas -Itests/emu/include -Itests/emu/gen -Iinclude -I$(CSRC)
tests/emu/gen/%.cpp: $(CSRC)/%.cu tests/emu/transform.py
	@mkdir -p tests/emu/gen
	python3 tests/emu/transform.py $< $@
tests/emu/gen/%.h: $(CSRC)/%.h tests/emu/transform.py
	@mkdir -p tests/emu/gen
	python3 tests/emu/transform.py $< $@
tests/emu/gen/%.cuh: $(CSRC)/%.cuh tests/emu/transform.py
	@mkdir -p tests/emu/gen
	python3 tests/emu/transform.py $< $@
$(EMU): $(EMU_GEN) $(EMU_HDRS) tests/emu/cuda_emu.cpp tests/emu/cuda_emu.h tests/emu/ldl_emu.cpp $(CPP_SRCS)
	$(CXX) $(EMU_FLAGS) -o $@ $(EMU_GEN) tests/emu/cuda_emu.cpp tests/emu/ldl_emu.cpp $(CPP_SRCS)
$(EMU_FULL): $(EMU_GEN) tests/emu/gen/ldl.cpp $(EMU_HDRS) tests/emu/cuda_emu.cpp tests/emu/cuda_emu.h $(CPP_SRCS)
	$(CXX) $(EMU_FLAGS) -o $@ $(EMU_GEN) tests/emu/gen/ldl.cpp tests/emu/cuda_emu.cpp $(CPP_SRCS)
emu: $(EMU) $(EMU_FULL)
all: $(EMU) $(EMU_FULL)
