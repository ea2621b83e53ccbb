# nvcc flags shared by the library (this directory's Makefile) and the device test harness
# (tests/cuda/Makefile), so that the harness runs field.cuh exactly as the kernels are compiled.
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 -lineinfo $(ARCH) -Xcompiler -fPIC -Xcompiler -Wall -Xcompiler -Wno-unknown-pragmas --expt-relaxed-constexpr
