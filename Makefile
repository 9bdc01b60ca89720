# Build of libdiscregrid_b200.so (sm_90a only: H100) and of the test-only oracle.
#   make lib     : discregrid_b200/lib/libdiscregrid_b200.so   (the product: CUDA kernels + C-ABI + host BVH builder)
#   make oracle  : oracle/liboracle.so (+ oracle/_ref when the reference sources are present, see oracle/Makefile)  -- test infrastructure
# -fmad=false / -ffp-contract=off are part of the numerical contract (bit-exact parity with the reference's
# non-FMA x86-64 build); dg_selftest() refuses to run a library built without them.
NVCC     ?= /usr/local/cuda/bin/nvcc
HOSTCXX  := $(shell command -v /usr/bin/g++ || echo g++)
ARCH     := -gencode arch=compute_90a,code=sm_90a
NVFLAGS  := $(ARCH) -ccbin $(HOSTCXX) -std=c++17 -O3 -lineinfo -fmad=false -Xcompiler -fPIC,-ffp-contract=off,-fvisibility=hidden
CXXFLAGS := -std=c++17 -O3 -fPIC -ffp-contract=off -fvisibility=hidden
SRC      := discregrid_b200/csrc
OBJ      := build/obj
LIB      := discregrid_b200/lib/libdiscregrid_b200.so
CU       := k1_sdf k2_interp k3_density k4_reduce k5_winding k6_isosurface k7_raycast k8_refit k9_mesh_raycast k10_distance_grad k11_field_grad k12_raycast_grad k13_isosurface_grad radix_sort dg_api
HDRS     := $(wildcard $(SRC)/*.h $(SRC)/*.cuh) include/discregrid_b200.h

all: lib cpp oracle
lib: $(LIB)

# C++ facade (cpp/include/Discregrid/*: the reference's class API over the C-ABI) -- the reference tools and a checker.
# Eigen3 is not installed in this image: cpp/eigen_min is used unless EIGEN3_INCLUDE_DIR points at the real one.
EIGEN3_INCLUDE_DIR ?= cpp/eigen_min
CPPBIN   := build/bin
CPPFLAGS := -std=c++11 -O2 -ffp-contract=off -I$(EIGEN3_INCLUDE_DIR) -Icpp/include -Iinclude
CPPLINK  := -Ldiscregrid_b200/lib -ldiscregrid_b200 -Wl,-rpath,'$$ORIGIN/../../discregrid_b200/lib'
CPPHDRS  := $(wildcard cpp/include/Discregrid/* cpp/include/Discregrid/*/*) include/discregrid_b200.h
cpp: $(CPPBIN)/GenerateSDF $(CPPBIN)/GenerateDensityMap $(CPPBIN)/GenerateVolumeMap $(CPPBIN)/liborcvolume.so ref_volume $(CPPBIN)/DiscreteFieldToBitmap $(CPPBIN)/DiscreteFieldToMesh $(CPPBIN)/facade_check $(CPPBIN)/bvh_host_check $(CPPBIN)/reduce_facade_check $(CPPBIN)/sort_replay_check $(CPPBIN)/fast_div_check $(CPPBIN)/libk1emu.so $(CPPBIN)/libk1emu_perlane.so $(CPPBIN)/libk1emu_band.so $(CPPBIN)/libk1emu_band_perlane.so $(CPPBIN)/libk23emu.so $(CPPBIN)/libk3vemu.so $(CPPBIN)/libk2hemu.so $(CPPBIN)/libk5emu.so $(CPPBIN)/libk8emu.so $(CPPBIN)/libk9emu.so $(CPPBIN)/libk9emu_nocull.so $(CPPBIN)/libk10emu.so $(CPPBIN)/libdgemu.so $(CPPBIN)/libk4emu.so $(CPPBIN)/device_function_check $(CPPBIN)/device_query_check $(CPPBIN)/hessian_check $(CPPBIN)/winding_check $(CPPBIN)/raycast_check $(CPPBIN)/refit_check $(CPPBIN)/mesh_raycast_check $(CPPBIN)/field_grad_check $(CPPBIN)/raycast_grad_check $(CPPBIN)/isosurface_grad_check $(CPPBIN)/liborctree.so
$(CPPBIN)/DiscreteFieldToBitmap: cpp/cmd/discrete_field_to_bitmap.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
$(CPPBIN)/DiscreteFieldToMesh: cpp/cmd/discrete_field_to_mesh.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
$(CPPBIN)/bvh_host_check: tests/cpp/bvh_host_check.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp $(SRC)/sort_replay.h $(SRC)/bvh_build.h
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CXXFLAGS) -fvisibility=default tests/cpp/bvh_host_check.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp -o $@ -lpthread
# test libraries: the K1 translation unit (kernels + launchers) compiled for the CPU by tests/emu -- the product's build (packet walk)
# and the per-lane node loop (K1_PACKET=0), the independent walk the packet walk is compared against
K1EMU_SRC := tests/emu/k1_emu.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
K1EMU_DEP := $(K1EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k1_sdf.cu $(HDRS)
CUDA_INC  ?= /usr/local/cuda/include
$(CPPBIN)/libk1emu.so: $(K1EMU_DEP)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K1EMU_SRC) -o $@ -lpthread
$(CPPBIN)/libk1emu_perlane.so: $(K1EMU_DEP)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -DK1_PACKET=0 -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K1EMU_SRC) -o $@ -lpthread
# the narrow-band launcher (classifier + band node loop) on top of the same TU: packet walk (default) and per-lane walk
K1BAND_SRC := tests/emu/k1_band_emu.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
$(CPPBIN)/libk1emu_band.so: $(K1EMU_DEP) tests/emu/k1_band_emu.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K1BAND_SRC) -o $@ -lpthread
$(CPPBIN)/libk1emu_band_perlane.so: $(K1EMU_DEP) tests/emu/k1_band_emu.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -DK1_PACKET=0 -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K1BAND_SRC) -o $@ -lpthread
K23EMU_SRC := tests/emu/k2_emu.cpp tests/emu/k3_emu.cpp
K23EMU_DEP := $(K23EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k2_interp.cu $(SRC)/k3_density.cu $(HDRS)
$(CPPBIN)/libk23emu.so: $(K23EMU_DEP)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K23EMU_SRC) -o $@ -lpthread
# the same with the volume map exposed (emu_volume_map, tests/emu/k3_volume_emu.cpp)
$(CPPBIN)/libk3vemu.so: $(K23EMU_DEP) tests/emu/k3_volume_emu.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) tests/emu/k2_emu.cpp tests/emu/k3_volume_emu.cpp -o $@ -lpthread
# the same with K2's Hessian mode exposed (emu_interpolate_hessian)
K2HEMU_SRC := tests/emu/k2_emu.cpp tests/emu/k2_hessian_emu.cpp
$(CPPBIN)/libk2hemu.so: $(K23EMU_DEP) tests/emu/k2_hessian_emu.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K2HEMU_SRC) -o $@ -lpthread
# the winding-number TU (k5_winding.cu: atan2, records, walk) with a small surface for tests/test_winding_emulated.py
K5EMU_SRC := tests/emu/k5_emu.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
$(CPPBIN)/libk5emu.so: $(K5EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k5_winding.cu $(HDRS)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K5EMU_SRC) -o $@ -lpthread
# the refit TU (k8_refit.cu: bounds, leaf, pseudonormal, sum, radius and packing passes) with a small surface for tests/test_refit_emulated.py
K8EMU_SRC := tests/emu/k8_emu.cpp tests/emu/k5_emu.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
$(CPPBIN)/libk8emu.so: $(K8EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k8_refit.cu $(SRC)/k5_winding.cu $(HDRS)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K8EMU_SRC) -o $@ -lpthread
# the mesh ray-cast TU (k9_mesh_raycast.cu) with a small surface for tests/test_mesh_raycast_emulated.py, with culling on (the product's build)
# and compiled out (K9_CULL=0), so that the culled walk is checked against the plain one
K9EMU_SRC := tests/emu/k9_emu.cpp tests/emu/k5_emu.cpp $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
K9EMU_DEP := $(K9EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k9_mesh_raycast.cu $(SRC)/k5_winding.cu $(HDRS)
$(CPPBIN)/libk9emu.so: $(K9EMU_DEP)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -DK9_EMU_SURFACE=1 -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K9EMU_SRC) -o $@ -lpthread
$(CPPBIN)/libk9emu_nocull.so: $(K9EMU_DEP)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -DK9_EMU_SURFACE=1 -DK9_CULL=0 -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K9EMU_SRC) -o $@ -lpthread
# the distance-gradient and radix-sort TUs (k10_distance_grad.cu, radix_sort.cu) with a small surface for tests/test_mesh_distance_grad_emulated.py
$(CPPBIN)/libk10emu.so: tests/emu/k10_emu.cpp tests/emu/cudart_stub.cpp tests/emu/cuda_emu.h $(SRC)/k10_distance_grad.cu $(SRC)/radix_sort.cu $(HDRS)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -Wl,-Bsymbolic -DK10_EMU_SURFACE=1 -I$(CUDA_INC) -Itests/emu -I$(SRC) tests/emu/k10_emu.cpp tests/emu/cudart_stub.cpp -o $@ -lpthread
# test library: the WHOLE product library with every kernel emulated and the CUDA runtime stubbed on host memory -- lets the Python-level
# and tool-level `-m gpu` tests be rehearsed on the CPU (tests/test_gpu_rehearsal.py); never loaded by the product
DGEMU_SRC := tests/emu/dgapi_emu.cpp tests/emu/k1_emu.cpp tests/emu/k2_emu.cpp tests/emu/k3_emu.cpp tests/emu/k4_emu.cpp tests/emu/k5_emu.cpp tests/emu/k6_emu.cpp tests/emu/k7_emu.cpp tests/emu/k8_emu.cpp tests/emu/k9_emu.cpp tests/emu/k10_emu.cpp tests/emu/k11_emu.cpp tests/emu/k12_emu.cpp tests/emu/k13_emu.cpp tests/emu/cudart_stub.cpp \
             $(SRC)/bvh_build.cpp $(SRC)/host_threads.cpp $(SRC)/reduce_field.cpp $(SRC)/obj_reader.cpp $(SRC)/sort_replay.cpp
$(CPPBIN)/libdgemu.so: $(DGEMU_SRC) tests/emu/cuda_emu.h $(wildcard $(SRC)/*.cu) $(HDRS)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -Wl,-Bsymbolic -Wno-subobject-linkage -I$(CUDA_INC) -Itests/emu -I$(SRC) -Iinclude $(DGEMU_SRC) -o $@ -lpthread
# test library: the device swap walk of k4_reduce.cu (emulated) next to the serial host walk of reduce_field.cpp it replaces
K4EMU_SRC := tests/emu/k4_walk_emu.cpp tests/emu/cudart_stub.cpp $(SRC)/reduce_field.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp
$(CPPBIN)/libk4emu.so: $(K4EMU_SRC) tests/emu/cuda_emu.h $(SRC)/k4_reduce.cu $(HDRS)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++17 -O2 -ffp-contract=off -fPIC -shared -Wl,-Bsymbolic -I$(CUDA_INC) -Itests/emu -I$(SRC) $(K4EMU_SRC) -o $@ -lpthread
# test binary: the reciprocal-based exact division of fast_div.h against '/' (brute force)
$(CPPBIN)/fast_div_check: tests/cpp/fast_div_check.cpp $(SRC)/fast_div.h $(SRC)/dg_device.cuh
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CXXFLAGS) -I$(SRC) tests/cpp/fast_div_check.cpp -o $@
# test binary: the threaded std::sort replay of reduce_field.cpp against std::sort (ties, depth exhaustion)
$(CPPBIN)/sort_replay_check: tests/cpp/sort_replay_check.cpp $(SRC)/reduce_field.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp $(SRC)/sort_replay.h $(SRC)/reduce_field.h $(SRC)/dg_device.cuh
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CXXFLAGS) -fvisibility=default -I$(SRC) tests/cpp/sort_replay_check.cpp $(SRC)/reduce_field.cpp $(SRC)/host_threads.cpp $(SRC)/sort_replay.cpp -o $@ -lpthread
# test binary: the facade's reduceField with dg_node_positions interposed by the oracle (runs without a GPU)
$(CPPBIN)/reduce_facade_check: tests/cpp/reduce_facade_check.cpp $(CPPHDRS) $(LIB) oracle/liboracle.so
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK) -Loracle -loracle -Wl,-rpath,'$$ORIGIN/../../oracle'
# test binary: the facade's device callbacks; they move data with the CUDA runtime (static, as the library links it)
CUDA_LIB ?= /usr/local/cuda/lib64
$(CPPBIN)/device_function_check: tests/cpp/device_function_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test binary: the facade's reduced calls feed interpolate from the kept handle; it defines its own dg_field_create, which refuses
$(CPPBIN)/device_query_check: tests/cpp/device_query_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
# test binary: the facade's batched Hessian overload on a grid file, for comparison with the Python route
$(CPPBIN)/hessian_check: tests/cpp/hessian_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
# test binary: the facade's sign mode (setSignMode, winding_number, signed_distance in the winding mode) on a mesh file
$(CPPBIN)/winding_check: tests/cpp/winding_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
# test binary: the facade's batched raycast on a grid file, for comparison with the Python route
$(CPPBIN)/raycast_check: tests/cpp/raycast_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
# test binary: the facade's refit (host vector and device pointer), for comparison with the Python route
$(CPPBIN)/refit_check: tests/cpp/refit_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test binary: the facade's mesh raycast (host arrays and device pointers), for comparison with the Python route
$(CPPBIN)/mesh_raycast_check: tests/cpp/mesh_raycast_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test binary: the facade's trainable field (setNodesDevice, interpolate_vjp on device pointers), for comparison with the Python route
$(CPPBIN)/field_grad_check: tests/cpp/field_grad_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test binary: the facade's ray-cast gradients (raycast_vjp of the mesh and of the grid on device pointers), for comparison with the Python route
$(CPPBIN)/raycast_grad_check: tests/cpp/raycast_grad_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test binary: the facade's level-set gradient (isosurface with edge ids, isosurface_vjp on device pointers), for comparison with the Python route
$(CPPBIN)/isosurface_grad_check: tests/cpp/isosurface_grad_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) -I$(CUDA_INC) $< -o $@ $(CPPLINK) -L$(CUDA_LIB) -lcudart_static -ldl -lrt -lpthread
# test library: the oracle with a given tree and given pseudonormals (the reference's query rule over a refit mesh's records)
$(CPPBIN)/liborctree.so: tests/cpp/oracle_from_tree.cpp oracle/dg_oracle.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++11 -O3 -DNDEBUG -fopenmp -ffp-contract=off -fPIC -shared $< -o $@
# test library: the oracle plus the volume map restated over its interpolate (orc_volume_map)
$(CPPBIN)/liborcvolume.so: tests/cpp/volume_oracle.cpp oracle/dg_oracle.cpp
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) -std=c++11 -O3 -DNDEBUG -fopenmp -ffp-contract=off -fPIC -shared $< -o $@
# the reference-side volume-map generator (oracle/ref_volume_map.cpp on the reference's own sources), when the reference is present
ref_volume:
	$(MAKE) -C oracle -f ref_volume.mk
oracle/liboracle.so:
	$(MAKE) -C oracle oracle
$(CPPBIN)/GenerateSDF: cpp/cmd/generate_sdf.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
$(CPPBIN)/GenerateDensityMap: cpp/cmd/generate_density_map.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
$(CPPBIN)/GenerateVolumeMap: cpp/cmd/generate_volume_map.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)
$(CPPBIN)/facade_check: cpp/cmd/facade_check.cpp $(CPPHDRS) $(LIB)
	@mkdir -p $(CPPBIN)
	$(HOSTCXX) $(CPPFLAGS) $< -o $@ $(CPPLINK)

$(OBJ)/%.o: $(SRC)/%.cu $(HDRS)
	@mkdir -p $(OBJ)
	$(NVCC) $(NVFLAGS) -c $< -o $@
$(OBJ)/%.o: $(SRC)/%.cpp $(HDRS)
	@mkdir -p $(OBJ)
	$(HOSTCXX) $(CXXFLAGS) -c $< -o $@

$(LIB): $(addprefix $(OBJ)/,$(addsuffix .o,$(CU))) $(OBJ)/bvh_build.o $(OBJ)/host_threads.o $(OBJ)/reduce_field.o $(OBJ)/obj_reader.o $(OBJ)/sort_replay.o
	@mkdir -p $(dir $(LIB))
	$(NVCC) $(ARCH) -ccbin $(HOSTCXX) -shared -o $@ $^ -Xlinker --exclude-libs=ALL

oracle:
	$(MAKE) -C oracle all

clean:
	rm -rf build $(LIB)
	$(MAKE) -C oracle clean
.PHONY: all lib cpp oracle ref_volume clean
