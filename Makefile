# Builds libdph_b200.so (sm_90a, H100 only) and the CPU oracle. `python -c "import __graft_entry__ as g; g.build()"` calls this.
NVCC ?= nvcc
ARCH := -gencode arch=compute_90a,code=sm_90a
NVFLAGS := -O3 -std=c++17 $(ARCH) -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr -Xptxas -v
CSRC := densephrases_b200/csrc
OBJDIR := build/obj
LIB := densephrases_b200/lib/libdph_b200.so
SRCS := $(wildcard $(CSRC)/*.cu)
OBJS := $(patsubst $(CSRC)/%.cu,$(OBJDIR)/%.o,$(SRCS))
HDRS := $(wildcard $(CSRC)/*.cuh) include/dph_b200.h

all: $(LIB) oracle

$(OBJDIR)/%.o: $(CSRC)/%.cu $(HDRS)
	@mkdir -p $(OBJDIR)
	$(NVCC) $(NVFLAGS) -c $< -o $@ 2> $(OBJDIR)/$*.ptxas.log || (cat $(OBJDIR)/$*.ptxas.log; exit 1)

$(LIB): $(OBJS)
	@mkdir -p densephrases_b200/lib
	$(NVCC) $(ARCH) -shared -o $@ $(OBJS) -lcudart

oracle: oracle/libivfpq_ref.so oracle/libencode_ref.so oracle/libremove_ref.so oracle/libtrain_ref.so oracle/libfilter_ref.so
oracle/libivfpq_ref.so: oracle/ivfpq_ref.c
	gcc -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared -fvisibility=hidden -o $@ $< -lm
oracle/libencode_ref.so: oracle/encode_ref.c oracle/ivfpq_ref.c
	gcc -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared -fvisibility=hidden -o $@ $< -lm
oracle/libremove_ref.so: oracle/remove_ref.c
	gcc -O3 -fPIC -shared -fvisibility=hidden -o $@ $<
oracle/libtrain_ref.so: oracle/train_ref.c oracle/ivfpq_ref.c
	gcc -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared -fvisibility=hidden -o $@ $< -lm

oracle/libfilter_ref.so: oracle/filter_ref.c oracle/ivfpq_ref.c
	gcc -O3 -march=x86-64-v3 -ffp-contract=off -fno-fast-math -fopenmp -fPIC -shared -fvisibility=hidden -o $@ $< -lm

clean:
	rm -rf build $(LIB) oracle/libivfpq_ref.so oracle/libencode_ref.so oracle/libremove_ref.so oracle/libtrain_ref.so oracle/libfilter_ref.so
.PHONY: all oracle clean
