# oracle/fxsynth.mk -- builds the end-to-end checker of a traced Synth that overrides processVector (TEST
# INFRASTRUCTURE ONLY), with the flags of oracle/Makefile (included for REF, REF_FLAGS and E2S_SRC):
#
#   _ref/libmlfxsynth.so  G complete reference AudioContext + Synth objects running tests/cpp/fx_synth_body.h
#                         (oracle/ref/mlfxsynth.cpp), compiled in place with the reference's MLAudioContext.cpp,
#                         MLValue.cpp and EventsToSignals sources.  Only where the reference tree exists; the built
#                         .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/fxsynth.mk fxsynth-ref
FXSYNTH_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(FXSYNTH_HERE)Makefile

fxsynth-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(FXSYNTH_HERE)fxsynth.mk $(FXSYNTH_HERE)_ref/libmlfxsynth.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(FXSYNTH_HERE)_ref/libmlfxsynth.so: $(FXSYNTH_HERE)ref/mlfxsynth.cpp $(FXSYNTH_HERE)../tests/cpp/fx_synth_body.h $(INC)/mlb200.h
	mkdir -p $(FXSYNTH_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(E2S_SRC) $(REF)/source/app/MLValue.cpp -lpthread

.PHONY: fxsynth-ref
