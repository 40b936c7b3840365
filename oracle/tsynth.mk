# oracle/tsynth.mk -- builds the end-to-end checker of mlb::tr::TracedSynth (TEST INFRASTRUCTURE ONLY), with the
# flags of oracle/Makefile (included for REF, REF_FLAGS and E2S_SRC):
#
#   _ref/libmltsynth.so   G complete reference AudioContext + Synth objects running tests/cpp/synth_body.h
#                         (oracle/ref/mltsynth.cpp), compiled in place with the reference's MLAudioContext.cpp,
#                         MLValue.cpp and EventsToSignals sources.  Only where the reference tree exists; the built
#                         .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/tsynth.mk tsynth-ref
TSYNTH_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(TSYNTH_HERE)Makefile

tsynth-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(TSYNTH_HERE)tsynth.mk $(TSYNTH_HERE)_ref/libmltsynth.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(TSYNTH_HERE)_ref/libmltsynth.so: $(TSYNTH_HERE)ref/mltsynth.cpp $(TSYNTH_HERE)../tests/cpp/synth_body.h $(INC)/mlb200.h
	mkdir -p $(TSYNTH_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(E2S_SRC) $(REF)/source/app/MLValue.cpp -lpthread

.PHONY: tsynth-ref
