# Builds libgf_b200.so (sm_90a, H100) in-tree.  `python -c "import __graft_entry__ as g; g.build()"` calls this.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
CSRC := ground_fusion_b200/csrc
OUT  := ground_fusion_b200/libgf_b200.so
YOLO_OUT := ground_fusion_b200/libgf_yolo.so
# -fmad=false: the front end is bit-exact with OpenCV's separately-rounded float ops (FMA only where written)
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden -fmad=false
SRCS := $(wildcard $(CSRC)/*.cu)
HDRS := $(wildcard $(CSRC)/*.cuh) $(CSRC)/gm_math.h include/gf_b200.h

all: $(OUT) $(YOLO_OUT) oracle

# front end: -fmad=false (bit-exact with OpenCV's separately-rounded float ops; FMA only where written)
# back end: default FMA contraction (parity is 1e-6 m against an FP64 oracle, not bit-exactness)
BUILD := ground_fusion_b200/csrc/_obj
$(BUILD)/fe_tracker.o: $(CSRC)/fe_tracker.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(NVFLAGS) -dc -o $@ $< -Xptxas -v 2> build_ptxas_fe.log || (cat build_ptxas_fe.log; false)
$(BUILD)/ba_solver.o: $(CSRC)/ba_solver.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -dc -o $@ $< -Xptxas -v 2> build_ptxas_ba.log || (cat build_ptxas_ba.log; false)
$(BUILD)/fm_kernels.o: $(CSRC)/fm_kernels.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -dc -o $@ $<
# landmark table: the flags of fm_kernels.o, whose arithmetic (fm_device.cuh) it shares bit for bit
$(BUILD)/fm_window.o: $(CSRC)/fm_window.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -dc -o $@ $< -Xptxas -v 2> build_ptxas_fmw.log || (cat build_ptxas_fmw.log; false)
# dense map: -fmad=false (bit-exact with oracle/dm_oracle.c, built with -ffp-contract=off)
$(BUILD)/dm_map.o: $(CSRC)/dm_map.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(NVFLAGS) -dc -o $@ $< -Xptxas -v 2> build_ptxas_dm.log || (cat build_ptxas_dm.log; false)
# occupancy grid: -fmad=false (bit-exact with oracle/gm_oracle.c's shared mode, built with -ffp-contract=off)
$(BUILD)/gm_grid.o: $(CSRC)/gm_grid.cu $(HDRS)
	@mkdir -p $(BUILD); $(NVCC) $(NVFLAGS) -dc -o $@ $< -Xptxas -v 2> build_ptxas_gm.log || (cat build_ptxas_gm.log; false)
# the detector's entry points in libgf_b200.so: host-only forwarders that open libgf_yolo.so on first use (no device code)
$(BUILD)/yolo_forward.o: $(CSRC)/yolo_forward.cpp include/gf_b200.h
	@mkdir -p $(BUILD); g++ -std=c++17 -O2 -fPIC -fvisibility=hidden -Wall -c -o $@ $<
$(OUT): $(BUILD)/fe_tracker.o $(BUILD)/ba_solver.o $(BUILD)/fm_kernels.o $(BUILD)/fm_window.o $(BUILD)/dm_map.o $(BUILD)/gm_grid.o $(BUILD)/yolo_forward.o
	$(NVCC) $(ARCH) -shared -o $@ $^ -ldl
	@cat build_ptxas_fe.log build_ptxas_ba.log build_ptxas_dm.log build_ptxas_gm.log build_ptxas_fmw.log > build_ptxas.log
# YOLO detector, its own library (the tracker / estimator library does not carry its device code): -fmad=false (bit-exact
# with darknet's CPU build, compiled with -ffp-contract=off by oracle/darknet.mk)
$(BUILD)/yolo_detector.o: $(CSRC)/yolo_detector.cu $(HDRS) $(CSRC)/yolo_cfg.cuh $(CSRC)/yolo_kernels.cuh
	@mkdir -p $(BUILD); $(NVCC) $(NVFLAGS) -c -o $@ $< -Xptxas -v 2> build_ptxas_yolo.log || (cat build_ptxas_yolo.log; false)
$(YOLO_OUT): $(BUILD)/yolo_detector.o
	$(NVCC) $(ARCH) -shared -o $@ $^

oracle: oracle/_build/libgf_oracle_dm.so oracle/_build/libgf_oracle_gm.so
	$(MAKE) -C oracle
	$(MAKE) -C oracle -f darknet.mk
	$(MAKE) -C oracle -f yolo_heads.mk
# the dense map's sequential restatement (tests and tools/bench_dense_map.py only): -O3 -ffp-contract=off as oracle/Makefile's
# libgf_oracle_ba.so, plus -msse2 -mfpmath=sse as its libgf_oracle_fe.so
oracle/_build/libgf_oracle_dm.so: oracle/dm_oracle.c
	@mkdir -p oracle/_build; gcc -O3 -ffp-contract=off -msse2 -mfpmath=sse -shared -fPIC -o $@ $< -lm
# the occupancy grid's sequential restatement, built like libgf_oracle_dm.so; it includes the kernel's shared log / exp
oracle/_build/libgf_oracle_gm.so: oracle/gm_oracle.c $(CSRC)/gm_math.h
	@mkdir -p oracle/_build; gcc -O3 -ffp-contract=off -msse2 -mfpmath=sse -shared -fPIC -o $@ $< -lm

# development aid: the same library with the clock64() phase counters compiled in (GF_B200_LIB=... selects it)
profile: $(SRCS) $(HDRS) $(BUILD)/fm_kernels.o $(BUILD)/fm_window.o $(BUILD)/dm_map.o $(BUILD)/gm_grid.o
	@mkdir -p $(BUILD)
	$(NVCC) $(NVFLAGS) -DGF_PROFILE -dc -o $(BUILD)/fe_tracker_prof.o $(CSRC)/fe_tracker.cu
	$(NVCC) $(filter-out -fmad=false,$(NVFLAGS)) -DGF_PROFILE -dc -o $(BUILD)/ba_solver_prof.o $(CSRC)/ba_solver.cu
	$(NVCC) $(ARCH) -shared -o ground_fusion_b200/libgf_b200_prof.so $(BUILD)/fe_tracker_prof.o $(BUILD)/ba_solver_prof.o $(BUILD)/fm_kernels.o $(BUILD)/fm_window.o $(BUILD)/dm_map.o $(BUILD)/gm_grid.o

clean:
	rm -f $(OUT) $(YOLO_OUT) build_ptxas.log build_ptxas_yolo.log; $(MAKE) -C oracle clean
.PHONY: all oracle clean profile
