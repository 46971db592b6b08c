# TEST INFRASTRUCTURE ONLY.  The reference's general-purpose hashes and proof of work for one reference build of
# oracle/Makefile, as an add-on next to it and to poseidon2.mk (whose libicicle_hash.so already holds the Keccak / SHA3 /
# Blake2s / Blake3 frontends and their dispatchers):
#
#   make -C oracle -f hash.mk hash CURVE=bn254 ID=1        (after `make ref` and `make -f poseidon2.mk poseidon2`)
#     -> _ref/<name>/libicicle_pow.so      : the PoW frontend (proof_of_work / proof_of_work_verify and their dispatchers)
#     -> _ref/<name>/libicicle_hash_cpu.so : the CPU backends of Keccak / SHA3, Blake2s, Blake3 and PoW, registered for "CPU"
#
# Source lists transcribed from icicle/cmake/hash.cmake:7-15 (src/hash/pow.cpp) and icicle/backend/cpu/CMakeLists.txt:84-92
# (the CPU backends).  Upstream links all of them into libicicle_hash; here they are libraries of their own, so that the
# libraries oracle/Makefile, poseidon2.mk and merkle.mk build stay exactly what they build.
include Makefile

POW_SRCS      := src/hash/pow.cpp
HASH_CPU_SRCS := backend/cpu/src/hash/cpu_keccak.cpp backend/cpu/src/hash/cpu_blake2s.cpp backend/cpu/src/hash/cpu_blake3.cpp \
                 backend/cpu/src/hash/cpu_pow.cpp
HASH_CPU_CSRCS := backend/cpu/src/hash/blake3.c backend/cpu/src/hash/blake3_dispatch.c backend/cpu/src/hash/blake3_portable.c
pow_objs      := $(patsubst %.cpp,$(O)/pow/%.o,$(POW_SRCS))
hash_cpu_objs := $(patsubst %.cpp,$(O)/hash_cpu/%.o,$(HASH_CPU_SRCS)) $(patsubst %.c,$(O)/hash_cpu/%.o,$(HASH_CPU_CSRCS))

.PHONY: hash
hash: $(D)/libicicle_pow.so $(D)/libicicle_hash_cpu.so

$(O)/pow/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(O)/hash_cpu/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@
$(O)/hash_cpu/%.o: $(SRC)/%.c
	@mkdir -p $(dir $@)
	$(CC) -O3 -DNDEBUG -fPIC -w -c $< -o $@

$(D)/libicicle_pow.so: $(pow_objs) $(D)/libicicle_device.so
	$(CXX) -shared -o $@ $(pow_objs) -L$(D) -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
$(D)/libicicle_hash_cpu.so: $(hash_cpu_objs) $(D)/libicicle_hash.so $(D)/libicicle_pow.so $(D)/libicicle_device.so
	$(CXX) -shared -o $@ $(hash_cpu_objs) -L$(D) -licicle_hash -licicle_pow -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
