# TEST INFRASTRUCTURE ONLY.  The reference's Merkle tree for one reference build of oracle/Makefile, as an add-on next to it
# and to poseidon2.mk (whose libicicle_hash.so it links):
#
#   make -C oracle -f merkle.mk merkle CURVE=bn254 ID=1        (after `make ref` and `make -f poseidon2.mk poseidon2`)
#     -> _ref/<name>/libicicle_merkle.so : the Merkle-tree frontend (icicle_merkle_tree_* / icicle_merkle_proof_*, the
#        merkle_tree_factory dispatcher) and the CPU tree (CPUMerkleTreeBackend, registered for "CPU")
#
# Source lists transcribed from icicle/cmake/hash.cmake:9-17 (frontend) and icicle/backend/cpu/CMakeLists.txt:84-92 (CPU
# tree).  Upstream links them into libicicle_hash; here they are a library of their own, so that the libraries
# oracle/Makefile and poseidon2.mk build stay exactly what they build.
include Makefile

MERKLE_SRCS := src/hash/merkle_tree.cpp src/hash/merkle_c_api.cpp backend/cpu/src/hash/cpu_merkle_tree.cpp
merkle_objs := $(patsubst %.cpp,$(O)/merkle/%.o,$(MERKLE_SRCS))

.PHONY: merkle
merkle: $(D)/libicicle_merkle.so

$(O)/merkle/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(D)/libicicle_merkle.so: $(merkle_objs) $(D)/libicicle_hash.so $(D)/libicicle_device.so
	$(CXX) -shared -o $@ $(merkle_objs) -L$(D) -licicle_hash -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
