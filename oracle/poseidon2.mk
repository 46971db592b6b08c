# TEST INFRASTRUCTURE ONLY.  The reference's Poseidon2 hash for one reference build of oracle/Makefile, as an add-on next to
# it; every family has POSEIDON2 in the reference's feature lists (icicle/cmake/features.cmake:5-19):
#
#   make -C oracle -f poseidon2.mk poseidon2 CURVE=bn254 ID=1        (after `make -C oracle ref CURVE=bn254 ID=1`)
#     -> _ref/<name>/libicicle_poseidon2_<name>.so : the Poseidon2 frontend (<name>_create_poseidon2_hasher, the
#        create_poseidon2 dispatcher) and its CPU backend, compiled with the build's defines plus -DPOSEIDON2=ON
#     -> _ref/<name>/libicicle_hash.so            : icicle_hasher_hash / _output_size / _delete
#
# Source lists transcribed from icicle/cmake/target_editor.cmake:99-105 (frontend), icicle/backend/cpu/CMakeLists.txt:56-57
# (CPU backend) and icicle/cmake/hash.cmake:7-15 (the hash library; only its C API and the general-purpose hash factories it
# calls are needed here, no tree builders).  Upstream links the Poseidon2 sources into libicicle_field_<name>; here they are a
# library of their own, so that the libraries oracle/Makefile builds stay exactly what it builds.
include Makefile

P2_SRCS   := src/hash/poseidon2.cpp src/hash/poseidon2_c_api.cpp backend/cpu/src/hash/cpu_poseidon2.cpp
HASH_SRCS := src/hash/keccak.cpp src/hash/blake2s.cpp src/hash/blake3.cpp src/hash/hash_c_api.cpp
p2_objs   := $(patsubst %.cpp,$(O)/poseidon2/%.o,$(P2_SRCS))
hash_objs := $(patsubst %.cpp,$(O)/hash/%.o,$(HASH_SRCS))

.PHONY: poseidon2
poseidon2: $(D)/libicicle_poseidon2_$(NAME).so $(D)/libicicle_hash.so

$(O)/poseidon2/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(DEFS) -DPOSEIDON2=ON -c $< -o $@
$(O)/hash/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(D)/libicicle_poseidon2_$(NAME).so: $(p2_objs) $(D)/libicicle_field_$(NAME).so
	$(CXX) -shared -o $@ $(p2_objs) -L$(D) -licicle_field_$(NAME) -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
$(D)/libicicle_hash.so: $(hash_objs) $(D)/libicicle_device.so
	$(CXX) -shared -o $@ $(hash_objs) -L$(D) -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
