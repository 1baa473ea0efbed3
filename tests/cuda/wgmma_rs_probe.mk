# Builds the register-A wgmma known-answer program (run by tests/test_wgmma_rs_gpu.py), sm_90a only:
#   make -C tests/cuda -f wgmma_rs_probe.mk
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
CSRC := ../../nonrigid_nerf_b200/csrc

all: wgmma_rs_probe

wgmma_rs_probe: wgmma_rs_probe.cu $(CSRC)/sm90_ptx.cuh
	$(NVCC) $(ARCH) -O2 -std=c++17 -I$(CSRC) $< -o $@

clean:
	rm -f wgmma_rs_probe
