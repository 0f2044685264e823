# Test-infrastructure recipe (nothing here is shipped in the product path):
#
#   make -f oracle/ref_vis.mk REF=<upstream radfoam checkout>
#       -> oracle/_ref/libradfoam_ref_vis.so: ref_vis_abi.cu (a C-ABI shim around the reference's
#          Pipeline::trace_visualization), linked against oracle/_ref/libradfoam_ref.so, which `make -C oracle ref`
#          builds from the reference's own tracing TU.  Flags as in oracle/Makefile.  Skipped when REF is absent.
HERE     := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
REF      ?= $(abspath $(HERE)../../reference)
NVCC     ?= nvcc
REF_OUT  := $(HERE)_ref
ARCH     ?= -gencode arch=compute_90a,code=sm_90a

.PHONY: ref_vis
ref_vis:
	@if [ -n "$(REF)" ] && [ -f $(REF)/src/tracing/pipeline.h ] && [ -f $(REF_OUT)/libradfoam_ref.so ]; then \
	    $(NVCC) -std=c++17 -O3 -lineinfo $(ARCH) --extended-lambda --expt-relaxed-constexpr \
	        -Xcompiler -fPIC -shared -w \
	        -I$(HERE)eigen_shim -I$(REF)/external/include -I$(REF)/src \
	        -o $(REF_OUT)/libradfoam_ref_vis.so $(HERE)ref_vis_abi.cu \
	        -L$(REF_OUT) -lradfoam_ref -Xlinker -rpath,'$$ORIGIN' ; \
	else \
	    echo "oracle/ref_vis.mk: $(REF) or $(REF_OUT)/libradfoam_ref.so absent; keeping prebuilt libradfoam_ref_vis.so" ; \
	fi
