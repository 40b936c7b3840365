# oracle/synth.mk -- builds the two CPU checkers of kernel K10, the per-instrument output buses (TEST INFRASTRUCTURE
# ONLY), with the flags of oracle/Makefile (included for REF, REF_FLAGS, PORT_FLAGS and E2S_SRC):
#
#   _port/libmlport_bus.so  plain-C strict-order restatement (oracle/port/mlport_bus.c), anywhere, any bus size
#   _ref/libmlsynth.so      the reference's own Synth::processVector (oracle/ref/mlsynth.cpp), compiled in place with
#                           the reference's MLAudioContext.cpp, MLValue.cpp and the EventsToSignals sources.  Only
#                           where the reference tree exists; the built .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/synth.mk bus-port | synth-ref
SYNTH_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(SYNTH_HERE)Makefile

bus-port: $(SYNTH_HERE)_port/libmlport_bus.so

$(SYNTH_HERE)_port/libmlport_bus.so: $(SYNTH_HERE)port/mlport_bus.c $(INC)/mlb200.h
	mkdir -p $(SYNTH_HERE)_port
	$(CC) $(PORT_FLAGS) -o $@ $<

synth-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(SYNTH_HERE)synth.mk $(SYNTH_HERE)_ref/libmlsynth.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(SYNTH_HERE)_ref/libmlsynth.so: $(SYNTH_HERE)ref/mlsynth.cpp
	mkdir -p $(SYNTH_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(E2S_SRC) $(REF)/source/app/MLValue.cpp -lpthread

.PHONY: bus-port synth-ref
