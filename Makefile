# Build of libabpoa_b200.so (host C + sm_90a CUDA) and of the test-only oracle.
#   make            -> abpoa_b200/lib/libabpoa_b200.so
#   make oracle     -> oracle/libpoa_oracle.so (+ oracle/_ref/ when /root/reference exists)
NVCC    ?= /usr/local/cuda/bin/nvcc
CC      ?= gcc
CSRC    := abpoa_b200/csrc
OBJ     := build/obj
LIBDIR  := abpoa_b200/lib
LIB     := $(LIBDIR)/libabpoa_b200.so
ARCH    := -gencode arch=compute_90a,code=sm_90a
CFLAGS  := -O2 -g -Wall -Wextra -Wno-unused-parameter -fPIC -Iinclude -I$(CSRC) -std=gnu11 -pthread
NVFLAGS := $(KPROF) $(ARCH) -O3 -lineinfo -std=c++17 -Xcompiler -fPIC,-Wall,-pthread -Iinclude -I$(CSRC)

C_SRCS  := $(wildcard $(CSRC)/*.c)
CU_SRCS := $(wildcard $(CSRC)/*.cu)
OBJS    := $(patsubst $(CSRC)/%.c,$(OBJ)/%.o,$(C_SRCS)) $(patsubst $(CSRC)/%.cu,$(OBJ)/%.cu.o,$(CU_SRCS))

BIN     := abpoa_b200/bin/abpoa

.PHONY: all oracle clean kprof
all: $(LIB) $(BIN)

$(OBJ)/%.o: $(CSRC)/%.c $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.cuh) $(wildcard include/*.h)
	@mkdir -p $(OBJ)
	$(CC) $(CFLAGS) -c $< -o $@

$(OBJ)/%.cu.o: $(CSRC)/%.cu $(wildcard $(CSRC)/*.h) $(wildcard $(CSRC)/*.cuh) $(wildcard include/*.h)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -c $< -o $@

$(LIB): $(OBJS)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -Xlinker -Bsymbolic -lm -lpthread -lz

# the `abpoa` command line (reference src/abpoa.c) over the library
$(BIN): abpoa_b200/cli/abpoa_cli.c $(LIB) $(wildcard include/*.h)
	@mkdir -p abpoa_b200/bin
	$(CC) -O2 -g -Wall -Iinclude -o $@ $< -L$(LIBDIR) -labpoa_b200 -Wl,-rpath,'$$ORIGIN/../lib' -lm

# profiling build of the same library (per-phase cycle counters inside the DP kernels): abpoa_b200/lib/libabpoa_b200_kprof.so,
# selected at run time with ABPOA_B200_LIB=<path>
kprof:
	$(MAKE) OBJ=build/obj_kprof LIB=$(LIBDIR)/libabpoa_b200_kprof.so KPROF=-DPOA_KPROF $(LIBDIR)/libabpoa_b200_kprof.so

oracle:
	$(MAKE) -C oracle all

clean:
	rm -rf build $(LIB) $(BIN)
