# Builds hybvio_b200/libhybvio_b200.so (sm_90a only: H100) and the test oracles.
NVCC ?= /usr/local/cuda/bin/nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-Wno-unused-function -Xptxas -v $(if $(TIMING),-DHV_EKF_TIMING,)
CSRC := hybvio_b200/csrc
OBJ := build/obj
LIB := hybvio_b200/libhybvio_b200.so
CU := $(wildcard $(CSRC)/*.cu)
OBJS := $(patsubst $(CSRC)/%.cu,$(OBJ)/%.o,$(CU))

DRV := hybvio_b200/libhv_e2e_driver.so
all: $(LIB) $(DRV) oracle

$(OBJ)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/hybvio_b200.h
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) $(if $(filter lk essential pose pnp triangulate,$*),--fmad=false,) -c $< -o $@ 2> $(OBJ)/$*.ptxas.log || (cat $(OBJ)/$*.ptxas.log; false)

$(LIB): $(OBJS)
	$(NVCC) $(ARCH) -shared -o $@ $^ -Xlinker --version-script=$(CSRC)/exports.map

# bench harness: native e2e caller of the C ABI (not part of the product library)
$(DRV): hybvio_b200/host/e2e_driver.cu include/hybvio_b200.h $(LIB)
	$(NVCC) $(ARCH) -O2 -std=c++17 -Xcompiler -fPIC -shared -o $@ $< -Lhybvio_b200 -lhybvio_b200 -Xlinker -rpath,'$$ORIGIN'

# instrumented copy (globaltimer phase marks in the EKF kernels) for tools/ekf_phases.py; never loaded by tests / bench
TOBJ := build/obj_timing
TLIB := hybvio_b200/libhybvio_b200_timing.so
$(TOBJ)/%.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.cuh) $(wildcard $(CSRC)/*.h) include/hybvio_b200.h
	@mkdir -p $(TOBJ)
	$(NVCC) $(NVFLAGS) -DHV_EKF_TIMING $(if $(filter lk essential pose pnp triangulate,$*),--fmad=false,) -c $< -o $@ 2> $(TOBJ)/$*.ptxas.log || (cat $(TOBJ)/$*.ptxas.log; false)
timing: $(patsubst $(CSRC)/%.cu,$(TOBJ)/%.o,$(CU))
	$(NVCC) $(ARCH) -shared -o $(TLIB) $^ -Xlinker --version-script=$(CSRC)/exports.map

oracle: oracle/libhv_oracle.so
oracle/libhv_oracle.so: $(wildcard oracle/*.c)
	gcc -O2 -ffp-contract=off -fPIC -shared -o $@ $^ -lm

ref:
	$(MAKE) -C oracle/ref_build -f Makefile.lk -j8

clean:
	rm -rf build $(LIB) $(DRV) oracle/libhv_oracle.so
.PHONY: all oracle ref clean timing
