# oracle/recorder.mk -- the reference's debug_mode report, for the recorder tests.  TEST INFRASTRUCTURE ONLY.
#
#   _ref/libfslic_ref_recorder.so: the UNMODIFIED reference, compiled from the sources where they lie under $(REF)
#                                  (never copied) with oracle/Makefile's flags, behind recorder_shim.cpp.  Only built
#                                  when REF names a checkout of Algy/fast-slic
#                                  (make -C oracle -f recorder.mk ref REF=/path/to/fast-slic).
REF ?= $(FSLIC_REFERENCE)
CXX = /usr/bin/g++
REF_SRCS = timer parallel fast-slic cca context context-impl lsc lsc-builder
REF_FLAGS = -std=c++11 -O3 -fopenmp -fPIC -DUSE_AVX2 -mavx2 -mfma -w
OBJ = _ref/recorder

ref:
	@if [ -n "$(REF)" ] && [ -d "$(REF)/src" ]; then $(MAKE) -f recorder.mk _ref/libfslic_ref_recorder.so; else echo "no fast-slic sources at REF='$(REF)': keeping prebuilt _ref"; fi

_ref/libfslic_ref_recorder.so: recorder_shim.cpp
	mkdir -p $(OBJ)
	for f in $(REF_SRCS); do $(CXX) $(REF_FLAGS) -c $(REF)/src/$$f.cpp -o $(OBJ)/$$f.o || exit 1; done
	$(CXX) $(REF_FLAGS) -I$(REF)/src -c recorder_shim.cpp -o $(OBJ)/recorder_shim.o
	$(CXX) -shared -fopenmp $(OBJ)/*.o -o _ref/libfslic_ref_recorder.so

clean:
	rm -rf $(OBJ) _ref/libfslic_ref_recorder.so
