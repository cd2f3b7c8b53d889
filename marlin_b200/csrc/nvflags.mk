# nvcc flags of libb2m.so, shared with tests/gpu/Makefile so that the kernel tests compile the product's
# headers exactly the way the product does.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := $(ARCH) -O3 -std=c++17 -lineinfo --extended-lambda -Xcompiler -fPIC -Xptxas -v
