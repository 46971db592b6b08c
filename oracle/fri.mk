# TEST INFRASTRUCTURE ONLY.  The reference's FRI for one reference build of oracle/Makefile, as an add-on next to it and to
# poseidon2.mk, merkle.mk and hash.mk (whose libraries it links):
#
#   make -C oracle -f fri.mk fri CURVE=bn254 ID=1     (after `make ref` and the poseidon2 / merkle / hash add-ons)
#     -> _ref/<name>/libicicle_fri_<name>.so : the FRI frontend (<name>_fri_merkle_tree_prove / _verify, <name>_fri_proof_*, the
#        fri_factory dispatcher; with EXT_FIELD also the <name>_extension_* entries) and the CPU prover (CpuFriBackend,
#        registered for "CPU"), compiled with the build's defines plus -DFRI=ON
#
# Source lists transcribed from icicle/cmake/target_editor.cmake:126-133 (handle_fri: src/fri/fri.cpp, src/fri/fri_c_api.cpp) and
# icicle/backend/cpu/CMakeLists.txt:62-63 (src/field/cpu_fri.cpp).  Upstream links them into libicicle_field_<name>;
# here they are a library of their own, so that the libraries oracle/Makefile and the other add-ons build stay exactly what
# they build.  The CPU prover reads the NTT domain CpuNttDomain<S>::s_ntt_domain, an inline static that the field library
# also defines: both are default-visibility unique symbols and this library links the field library, so the loader binds
# them to one object (the one <name>_ntt_init_domain fills).
include Makefile

FRI_SRCS := src/fri/fri.cpp src/fri/fri_c_api.cpp backend/cpu/src/field/cpu_fri.cpp
fri_objs := $(patsubst %.cpp,$(O)/fri/%.o,$(FRI_SRCS))

.PHONY: fri
fri: $(D)/libicicle_fri_$(NAME).so

$(O)/fri/%.o: $(SRC)/%.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) $(DEFS) -DFRI=ON -c $< -o $@

$(D)/libicicle_fri_$(NAME).so: $(fri_objs) $(D)/libicicle_field_$(NAME).so $(D)/libicicle_merkle.so $(D)/libicicle_pow.so $(D)/libicicle_hash.so
	$(CXX) -shared -o $@ $(fri_objs) -L$(D) -licicle_field_$(NAME) -licicle_merkle -licicle_pow -licicle_hash -licicle_device -Wl,-rpath,'$$ORIGIN' -pthread
