# oracle/ptime.mk -- builds the two CPU checkers of kernel K13, the host-transport beat phase of AudioContext
# (TEST INFRASTRUCTURE ONLY), with the flags of oracle/Makefile (included for REF, REF_FLAGS, PORT_FLAGS and E2S_SRC):
#
#   _port/libmlport_ptime.so  plain-C restatement fed by the CSR transport list (oracle/port/mlport_ptime.c), anywhere
#   _ref/libmlptime.so        one complete reference AudioContext per instrument (oracle/ref/mlptime.cpp), compiled
#                             in place with the reference's MLAudioContext.cpp, MLValue.cpp and EventsToSignals
#                             sources.  Only where the reference tree exists; the built .so travels with the other
#                             oracle/_ref libraries.
#
#   make -f oracle/ptime.mk ptime-port | ptime-ref
PTIME_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(PTIME_HERE)Makefile

ptime-port: $(PTIME_HERE)_port/libmlport_ptime.so

$(PTIME_HERE)_port/libmlport_ptime.so: $(PTIME_HERE)port/mlport_ptime.c $(INC)/mlb200.h
	mkdir -p $(PTIME_HERE)_port
	$(CC) $(PORT_FLAGS) -o $@ $< -lm

ptime-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(PTIME_HERE)ptime.mk $(PTIME_HERE)_ref/libmlptime.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(PTIME_HERE)_ref/libmlptime.so: $(PTIME_HERE)ref/mlptime.cpp $(INC)/mlb200.h
	mkdir -p $(PTIME_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(E2S_SRC) $(REF)/source/app/MLValue.cpp -lpthread

.PHONY: ptime-port ptime-ref
