# Builds the register-A wgmma known-answer program for N = 64 and the skip layer's two consumers of one set of fragments
# (run by tests/test_wgmma_rs64_gpu.py), sm_90a only:
#   make -C tests/cuda -f wgmma_rs64_probe.mk
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
CSRC := ../../nonrigid_nerf_b200/csrc

all: wgmma_rs64_probe

wgmma_rs64_probe: wgmma_rs64_probe.cu $(CSRC)/sm90_ptx.cuh
	$(NVCC) $(ARCH) -O2 -std=c++17 -I$(CSRC) $< -o $@

clean:
	rm -f wgmma_rs64_probe
