# Builds libgf_b200.so (sm_90a, H100) in-tree.  `python -c "import __graft_entry__ as g; g.build()"` calls this.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
CSRC := ground_fusion_b200/csrc
OUT  := ground_fusion_b200/libgf_b200.so
# -fmad=false: the front end is bit-exact with OpenCV's separately-rounded float ops (FMA only where written)
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden -fmad=false
SRCS := $(wildcard $(CSRC)/*.cu)
HDRS := $(wildcard $(CSRC)/*.cuh) include/gf_b200.h

all: $(OUT) oracle

# front end: -fmad=false (bit-exact with OpenCV's separately-rounded float ops; FMA only where written)
# back end: default FMA contraction (parity is 1e-6 m against an FP64 oracle, not bit-exactness)
BUILD := ground_fusion_b200/csrc/_obj
$(BUILD)/fe_tracker.o: $(CSRC)/fe_tracker.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(NVFLAGS) -dc -o $@ $< -Xptxas -v 2> build_ptxas_fe.log || (cat build_ptxas_fe.log; false)
$(BUILD)/ba_solver.o: $(CSRC)/ba_solver.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -dc -o $@ $< -Xptxas -v 2> build_ptxas_ba.log || (cat build_ptxas_ba.log; false)
$(BUILD)/fm_kernels.o: $(CSRC)/fm_kernels.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -dc -o $@ $<
$(OUT): $(BUILD)/fe_tracker.o $(BUILD)/ba_solver.o $(BUILD)/fm_kernels.o
	$(NVCC) $(ARCH) -shared -o $@ $^
	@cat build_ptxas_fe.log build_ptxas_ba.log > build_ptxas.log

oracle:
	$(MAKE) -C oracle

# development aid: the same library with the clock64() phase counters compiled in (GF_B200_LIB=... selects it)
profile: $(SRCS) $(HDRS) $(BUILD)/fm_kernels.o
	@mkdir -p $(BUILD)
	$(NVCC) $(NVFLAGS) -DGF_PROFILE -dc -o $(BUILD)/fe_tracker_prof.o $(CSRC)/fe_tracker.cu
	$(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -DGF_PROFILE -dc -o $(BUILD)/ba_solver_prof.o $(CSRC)/ba_solver.cu
	$(NVCC) $(ARCH) -shared -o ground_fusion_b200/libgf_b200_prof.so $(BUILD)/fe_tracker_prof.o $(BUILD)/ba_solver_prof.o $(BUILD)/fm_kernels.o

clean:
	rm -f $(OUT) build_ptxas.log; $(MAKE) -C oracle clean
.PHONY: all oracle clean profile
