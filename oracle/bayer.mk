# oracle/bayer.mk -- TEST INFRASTRUCTURE ONLY: the checkers of the BYR4 decode output, built beside those of Makefile with
# its compilers, flags and directories.
#
#  * liboracle_bayer.so        : the restated Bayer reconstruction (cfhd_oracle_bayer.c)
#  * _ref/libcfhd_ref_bayer.so : ref_probe_bayer.cpp, linked to _ref/libcfhd_ref.so (the unmodified reference)
#
#     make -C oracle -f bayer.mk bayer
include Makefile

.PHONY: bayer bayer_ref
bayer: liboracle_bayer.so bayer_ref

liboracle_bayer.so: cfhd_oracle_bayer.c cfhd_oracle_bayer.h
	$(CC) -O2 -fPIC -shared -Wall -o $@ cfhd_oracle_bayer.c

ifneq ($(wildcard $(REF)/Codec/spatial.c),)
bayer_ref: $(OUT)/libcfhd_ref_bayer.so
else
bayer_ref:
	@echo "oracle: $(REF) not present; using prebuilt $(OUT)/ if any"
endif

$(OBJ)/ref_probe_bayer.opp: ref_probe_bayer.cpp
	@mkdir -p $(dir $@)
	$(CXX) $(CXXFLAGS) -c $< -o $@

$(OUT)/libcfhd_ref_bayer.so: $(OBJ)/ref_probe_bayer.opp $(OUT)/libcfhd_ref.so
	$(CXX) -shared -o $@ $< -L$(OUT) -lcfhd_ref -Wl,-rpath,'$$ORIGIN'
