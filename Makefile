# b200mpi native build (sm_90a only). `make` builds everything in-tree; the
# built artefacts are git-ignored.
comma     := ,
NVCC      ?= /usr/local/cuda/bin/nvcc
CXX       ?= g++
ARCH      := -gencode arch=compute_90a,code=sm_90a
NVFLAGS   := -std=c++17 -O3 -lineinfo $(ARCH) -Xcompiler -fPIC,-Wall,-Wno-unused-function -Icsrc/include
CXXFLAGS  := -std=c++17 -O2 -fPIC -Wall -Icsrc/include
LIBDIR    := mpi_operator_b200/lib
BINDIR    := mpi_operator_b200/bin

RUNTIME_SRCS := csrc/kernels/collectives.cu csrc/kernels/adasum.cu csrc/kernels/bn_act.cu csrc/kernels/p2p.cu csrc/runtime/comm.cc csrc/runtime/rendezvous.cc
RUNTIME_HDRS := csrc/include/b200mpi.h csrc/kernels/device.cuh csrc/kernels/kernels.h csrc/runtime/rendezvous.h

all: $(LIBDIR)/libb200mpi.so $(LIBDIR)/libb200mpi_nccl.so $(LIBDIR)/libb200mpi_gemm.so native

# -Bsymbolic: the NCCL-ABI shim contains the same sources and is LD_PRELOADed into every rank by the node agent; without it
# the runtime's internal calls would bind to the preloaded copy while its entry points (looked up by handle) stay local,
# i.e. one call would run through two copies of the file-static state.
$(LIBDIR)/libb200mpi.so: $(RUNTIME_SRCS) $(RUNTIME_HDRS)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(NVFLAGS) -shared -x cu $(RUNTIME_SRCS) -o $@ -lrt -lpthread -Xlinker -Bsymbolic

$(LIBDIR)/libb200mpi_nccl.so: csrc/nccl_shim/nccl_shim.cu $(RUNTIME_SRCS) $(RUNTIME_HDRS)
	@mkdir -p $(LIBDIR)
	$(NVCC) $(NVFLAGS) -shared -x cu csrc/nccl_shim/nccl_shim.cu $(RUNTIME_SRCS) -o $@ -lrt -lpthread -ldl

# wgmma/TMA GEMM with fused BN statistics: a library of its own so that the experimental kernel cannot affect
# the validated runtime library
$(LIBDIR)/libb200mpi_gemm.so: csrc/kernels/gemm_bnstats.cu csrc/kernels/gemm_bnstats_logic.h csrc/include/b200mpi.h
	@mkdir -p $(LIBDIR)
	$(NVCC) $(NVFLAGS) -shared csrc/kernels/gemm_bnstats.cu -o $@

native: $(BINDIR)/mpirun $(LIBDIR)/libmpi.so $(LIBDIR)/libb200mpi_hvd.so $(BINDIR)/pi $(BINDIR)/pingpong

$(BINDIR)/mpirun: csrc/spawner/mpirun.cc
	@mkdir -p $(BINDIR)
	$(CXX) $(CXXFLAGS) -o $@ $<
	ln -sf mpirun $(BINDIR)/mpiexec
	ln -sf mpirun $(BINDIR)/mpiexec.hydra
	ln -sf mpirun $(BINDIR)/orterun
	printf '#!/bin/sh\nexec python -m mpi_operator_b200.cmd.horovodrun "$$@"\n' > $(BINDIR)/horovodrun && chmod +x $(BINDIR)/horovodrun

$(LIBDIR)/libmpi.so: csrc/mpi_shim/mpi_shim.cc csrc/mpi_shim/mpi_p2p.cc csrc/mpi_shim/mpi_comm.cc csrc/mpi_shim/mpi_internal.h csrc/mpi_shim/mpi.h csrc/runtime/rendezvous.cc csrc/runtime/rendezvous.h
	@mkdir -p $(LIBDIR) mpi_operator_b200/include
	$(CXX) $(CXXFLAGS) -shared -o $@ csrc/mpi_shim/mpi_shim.cc csrc/mpi_shim/mpi_p2p.cc csrc/mpi_shim/mpi_comm.cc csrc/runtime/rendezvous.cc -lrt -lpthread
	cp csrc/mpi_shim/mpi.h mpi_operator_b200/include/mpi.h

# Horovod-core equivalent: negotiation / fusion / response cache / timeline / stall inspector (host only, no CUDA link:
# the GPU executor calls libb200mpi.so and the process's cudart through function pointers)
HVD_SRCS := csrc/hvd_core/hvd_core.cc csrc/runtime/rendezvous.cc
$(LIBDIR)/libb200mpi_hvd.so: $(HVD_SRCS) csrc/hvd_core/hvd_core.h csrc/runtime/rendezvous.h
	@mkdir -p $(LIBDIR)
	$(CXX) $(CXXFLAGS) -Wextra -Wno-unused-parameter -shared -o $@ $(HVD_SRCS) -lrt -lpthread -ldl

$(BINDIR)/pi: examples/pi/pi.cc $(LIBDIR)/libmpi.so
	$(CXX) -std=c++17 -O2 -Impi_operator_b200/include -o $@ $< -L$(LIBDIR) -lmpi -Wl,-rpath,'$$ORIGIN/../lib'

$(BINDIR)/pingpong: examples/mpi-ring/pingpong.cc $(LIBDIR)/libmpi.so
	$(CXX) -std=c++17 -O2 -Impi_operator_b200/include -o $@ $< -L$(LIBDIR) -lmpi -Wl,-rpath,'$$ORIGIN/../lib'

sass: $(LIBDIR)/libb200mpi.so
	@mkdir -p profiles
	/usr/local/cuda/bin/cuobjdump -sass $(LIBDIR)/libb200mpi.so > profiles/libb200mpi.sass

clean:
	rm -rf $(LIBDIR)/*.so $(BINDIR)/*

# ---- developer targets (reference Makefile:64-98: fmt, vet, test, test_e2e, generate, verify-generate) ----
test:
	python -m pytest tests -x -q -m "not gpu"

test_gpu:
	python -m pytest tests -x -q -m gpu

test_e2e: all
	python -m mpi_operator_b200.cmd.mpijobctl run -f examples/pi/pi.yaml --fake-gpus 0

generate:
	python hack/generate.py

verify-generate:
	python hack/generate.py --verify

lint:
	python -m compileall -q mpi_operator_b200 tests bench.py __graft_entry__.py

sanitize: all
	tools/sanitize.sh

# Host-side runtime under the compiler sanitizers (SURVEY.md §5.2): launcher, shm rendezvous, libmpi shim.
SAN_CXX  ?= /usr/bin/g++
SAN_SRCS := csrc/mpi_shim/mpi_shim.cc csrc/mpi_shim/mpi_p2p.cc csrc/mpi_shim/mpi_comm.cc csrc/runtime/rendezvous.cc
define san_build
	@mkdir -p build/san/$(1)
	$(SAN_CXX) -std=c++17 -O1 -g -fno-omit-frame-pointer $(2) -Icsrc/include -o build/san/$(1)/mpirun csrc/spawner/mpirun.cc
	$(SAN_CXX) -std=c++17 -O1 -g -fno-omit-frame-pointer $(2) -Icsrc/include -Icsrc/mpi_shim -o build/san/$(1)/mpi_stress csrc/tests/mpi_stress.cc $(SAN_SRCS) -lrt -lpthread
	$(SAN_CXX) -std=c++17 -O1 -g -fno-omit-frame-pointer $(2) -Icsrc/include -Icsrc/mpi_shim -o build/san/$(1)/pi examples/pi/pi.cc $(SAN_SRCS) -lrt -lpthread
	$(SAN_CXX) -std=c++17 -O1 -g -fno-omit-frame-pointer $(2) -Icsrc/include -Icsrc/mpi_shim -o build/san/$(1)/mpi_p2p_test csrc/tests/mpi_p2p_test.cc $(SAN_SRCS) -lrt -lpthread
	$(SAN_CXX) -std=c++17 -O1 -g -fno-omit-frame-pointer $(2) -Icsrc/include -o build/san/$(1)/hvd_core_test csrc/tests/hvd_core_test.cc $(HVD_SRCS) -lrt -lpthread -ldl
endef

# negotiation / fusion / cache / join semantics of the hvdcore engine on 4 ranks (and 1, 3: odd world sizes)
test_hvd_core: native
	@mkdir -p build/san
	$(CXX) -std=c++17 -O2 -Wall -Icsrc/include -o build/san/hvd_core_test csrc/tests/hvd_core_test.cc $(HVD_SRCS) -lrt -lpthread -ldl
	$(BINDIR)/mpirun -n 4 build/san/hvd_core_test
	$(BINDIR)/mpirun -n 3 build/san/hvd_core_test
	$(BINDIR)/mpirun -n 1 build/san/hvd_core_test

# launch planning / counters of the runtime, checked on the host (no GPU): includes comm.cc, kernels come from the .so
test_comm_host: $(LIBDIR)/libb200mpi.so
	@mkdir -p build/san
	$(NVCC) -std=c++17 -O1 $(ARCH) -Icsrc/include -x cu csrc/tests/comm_host_test.cu -o build/san/comm_host_test -L$(LIBDIR) -lb200mpi -Xlinker -rpath,$(abspath $(LIBDIR)) -lrt -lpthread
	build/san/comm_host_test

# MPI point-to-point / v-collective semantics of the libmpi shim on 4 ranks
test_mpi_p2p: native
	@mkdir -p build/san
	$(CXX) -std=c++17 -O2 -Wall -Impi_operator_b200/include -o build/san/mpi_p2p_test csrc/tests/mpi_p2p_test.cc -L$(LIBDIR) -lmpi -Wl,-rpath,$(abspath $(LIBDIR))
	$(BINDIR)/mpirun -n 4 build/san/mpi_p2p_test
	$(BINDIR)/mpirun -n 5 build/san/mpi_p2p_test
	$(BINDIR)/mpirun -n 2 build/san/mpi_p2p_test
	$(BINDIR)/mpirun -n 1 build/san/mpi_p2p_test

# the point-to-point protocol of p2p.cu run with host threads instead of CTAs (same template, host platform)
test_p2p_protocol: $(LIBDIR)/libb200mpi.so
	@mkdir -p build/san
	$(NVCC) -std=c++17 -O1 $(ARCH) -Icsrc/include -Xcudafe --diag_suppress=20011,--diag_suppress=20014 -x cu csrc/tests/p2p_protocol_test.cu -o build/san/p2p_protocol_test -L$(LIBDIR) -lb200mpi -Xlinker -rpath,$(abspath $(LIBDIR)) -lrt -lpthread
	build/san/p2p_protocol_test

# host model of the wgmma GEMM's producer / consumer pipeline (shares gemm_bnstats_logic.h with the kernel)
test_gemm_model:
	@mkdir -p build/san
	$(CXX) -std=c++17 -O2 -Wall -o build/san/gemm_pipeline_model csrc/tests/gemm_pipeline_model.cc -lpthread
	build/san/gemm_pipeline_model

# hand-packed wgmma descriptor vs CuTe's (CUTLASS headers as shipped with the flashinfer wheel; pass CUTLASS_INC=... elsewhere)
CUTLASS_INC ?= $(shell python -c "import importlib.util,os;s=importlib.util.find_spec('flashinfer');print(os.path.join(os.path.dirname(s.origin),'data','cutlass','include'))" 2>/dev/null)
test_gmma_desc:
	@mkdir -p build/san
	$(NVCC) -std=c++17 -O1 $(ARCH) --expt-relaxed-constexpr -Icsrc/include -I$(CUTLASS_INC) -x cu csrc/tests/gmma_desc_test.cu -o build/san/gmma_desc_test
	build/san/gmma_desc_test 2>/dev/null

asan:
	$(call san_build,asan,-fsanitize=address$(comma)undefined -fno-sanitize-recover=undefined)
	ASAN_OPTIONS=detect_leaks=1:abort_on_error=0 build/san/asan/mpirun -n 4 build/san/asan/mpi_stress 200
	build/san/asan/mpirun -n 2 --tag-output build/san/asan/pi
	build/san/asan/mpirun -n 4 build/san/asan/mpi_p2p_test
	ASAN_OPTIONS=detect_leaks=1 build/san/asan/mpirun -n 4 build/san/asan/hvd_core_test

tsan:
	$(call san_build,tsan,-fsanitize=thread)
	TSAN_OPTIONS=halt_on_error=1 build/san/tsan/mpirun -n 4 build/san/tsan/mpi_stress 200
	build/san/tsan/mpirun -n 2 build/san/tsan/pi
	TSAN_OPTIONS=halt_on_error=1 build/san/tsan/mpirun -n 4 build/san/tsan/hvd_core_test
	# device protocols executed by host threads (same templates / shared logic as the kernels) under ThreadSanitizer:
	# every shared-memory, mailbox and flag access must be ordered by the barriers the kernels use
	$(SAN_CXX) -std=c++17 -O1 -g -fsanitize=thread -o build/san/tsan/gemm_pipeline_model csrc/tests/gemm_pipeline_model.cc -lpthread
	TSAN_OPTIONS=halt_on_error=1 build/san/tsan/gemm_pipeline_model
	$(NVCC) -ccbin $(SAN_CXX) -std=c++17 -O1 -g $(ARCH) -Icsrc/include -Xcudafe --diag_suppress=20011,--diag_suppress=20014 -Xcompiler -fsanitize=thread -x cu csrc/tests/p2p_protocol_test.cu -o build/san/tsan/p2p_protocol_test -L$(LIBDIR) -lb200mpi -Xlinker -rpath,$(abspath $(LIBDIR)) -lrt -lpthread -ltsan
	TSAN_OPTIONS=halt_on_error=1 build/san/tsan/p2p_protocol_test

.PHONY: all native sass clean test test_gpu test_e2e generate verify-generate lint sanitize asan tsan test_comm_host test_gmma_desc test_p2p_protocol test_gemm_model test_mpi_p2p test_hvd_core
