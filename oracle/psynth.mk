# oracle/psynth.mk -- builds the end-to-end checker of published signals of mlb::tr::TracedSynth (TEST INFRASTRUCTURE
# ONLY), with the flags of oracle/Makefile (included for REF, REF_FLAGS and E2S_SRC):
#
#   _ref/libmlpsynth.so   G complete reference AudioContext + Synth objects running tests/cpp/published_body.h
#                         (oracle/ref/mlpsynth.cpp), compiled in place with the reference's MLAudioContext.cpp,
#                         MLSignalProcessor.cpp, MLValue.cpp and EventsToSignals sources.  Only where the reference
#                         tree exists; the built .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/psynth.mk psynth-ref
PSYNTH_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(PSYNTH_HERE)Makefile

psynth-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(PSYNTH_HERE)psynth.mk $(PSYNTH_HERE)_ref/libmlpsynth.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(PSYNTH_HERE)_ref/libmlpsynth.so: $(PSYNTH_HERE)ref/mlpsynth.cpp $(PSYNTH_HERE)psynth.mk $(PSYNTH_HERE)../tests/cpp/published_body.h $(INC)/mlb200.h
	mkdir -p $(PSYNTH_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(REF)/source/app/MLSignalProcessor.cpp $(E2S_SRC) \
	  $(REF)/source/app/MLValue.cpp $(REF)/source/app/MLPath.cpp -lpthread

.PHONY: psynth-ref
