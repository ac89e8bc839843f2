# Builds the reference's own 2:4-sparse fp8 compressor and GEMM (CUTLASS 3 Sm90 sparse tensor-op code) in place
# from the reference tree into _ref/libref_sparse_f8.so. Test infrastructure only: the GPU tests and
# scripts/measure_fp8_sparse.py compare the engine's sparse path against it. Nothing is copied from the tree.
#
#   make -f ref_sparse.mk REF=<reference root> PY_INC="<torch include dirs> <python include>" TORCH_LIB=<torch/lib>
#
# The flags follow the reference's setup.py for its cutlass_90a extension. The dispatcher references all four
# dtype units, so all four are built (in parallel with make -j; the e4m3e4m3 unit alone takes minutes).
NVCC ?= /usr/local/cuda/bin/nvcc
REF ?= /root/reference
CSRC := $(REF)/torchao/csrc/cuda
OUT := _ref
LIB := $(OUT)/libref_sparse_f8.so

FLAGS := -std=c++17 -O3 -DNDEBUG -DUSE_CUDA -DTORCH_TARGET_VERSION=0x020b000000000000 \
         -gencode arch=compute_90a,code=sm_90a -DTORCHAO_USE_CUTLASS \
         -DBUILD_TO_SPARSE_SEMI_STRUCTURED_CUTLASS_SM9X -DBUILD_ROWWISE_SCALED_LINEAR_SPARSE_CUTLASS \
         -DCUTLASS_ENABLE_TENSOR_CORE_MMA=1 -DCUTLASS_DEBUG_TRACE_LEVEL=0 --expt-relaxed-constexpr \
         -I$(REF)/third_party/cutlass/include -I$(REF)/third_party/cutlass/tools/util/include -I$(CSRC) \
         $(addprefix -I,$(PY_INC)) -Xcompiler -fPIC

GEMM := $(CSRC)/rowwise_scaled_linear_sparse_cutlass/rowwise_scaled_linear_sparse_cutlass
SRCS := $(CSRC)/to_sparse_semi_structured_cutlass_sm9x/to_sparse_semi_structured_cutlass_sm9x_f8.cu \
        $(GEMM)_f8f8.cu $(GEMM)_e4m3e4m3.cu $(GEMM)_e4m3e5m2.cu $(GEMM)_e5m2e4m3.cu $(GEMM)_e5m2e5m2.cu
OBJS := $(addprefix $(OUT)/,$(notdir $(SRCS:.cu=.o)))
# every object also depends on the headers of both kernels and on this recipe
HDRS := $(CSRC)/to_sparse_semi_structured_cutlass_sm9x/to_sparse_semi_structured_cutlass_sm9x.cuh \
        $(GEMM).cuh $(wildcard $(GEMM)_*.h) ref_sparse.mk

all: $(LIB)

$(LIB): $(OBJS)
	$(NVCC) -shared -cudart shared -o $@ $^ -L$(TORCH_LIB) -ltorch -ltorch_cpu -ltorch_cuda -lc10 -lc10_cuda -lcuda

$(OUT)/%.o: $(CSRC)/to_sparse_semi_structured_cutlass_sm9x/%.cu $(HDRS)
	@mkdir -p $(OUT)
	$(NVCC) $(FLAGS) -c $< -o $@

$(OUT)/%.o: $(CSRC)/rowwise_scaled_linear_sparse_cutlass/%.cu $(HDRS)
	@mkdir -p $(OUT)
	$(NVCC) $(FLAGS) -c $< -o $@

.PHONY: all
