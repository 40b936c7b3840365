# oracle/ctrl.mk -- builds the two CPU checkers of kernel K11, the smoothed MIDI controllers (TEST INFRASTRUCTURE
# ONLY), with the flags of oracle/Makefile (included for REF, REF_FLAGS, PORT_FLAGS and E2S_SRC):
#
#   _port/libmlport_ctrl.so  plain-C restatement fed by the CSR change list (oracle/port/mlport_ctrl.c), anywhere
#   _ref/libmlctrl.so        one complete reference EventsToSignals per instrument (oracle/ref/mlctrl.cpp), compiled
#                            in place with the reference's EventsToSignals sources.  Only where the reference tree
#                            exists; the built .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/ctrl.mk ctrl-port | ctrl-ref
CTRL_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(CTRL_HERE)Makefile

ctrl-port: $(CTRL_HERE)_port/libmlport_ctrl.so

$(CTRL_HERE)_port/libmlport_ctrl.so: $(CTRL_HERE)port/mlport_ctrl.c $(INC)/mlb200.h
	mkdir -p $(CTRL_HERE)_port
	$(CC) $(PORT_FLAGS) -o $@ $<

ctrl-ref:
	@if [ -d "$(REF)/source/DSP" ]; then $(MAKE) -f $(CTRL_HERE)ctrl.mk $(CTRL_HERE)_ref/libmlctrl.so; \
	else echo "reference tree not present at $(REF): keeping prebuilt oracle/_ref (if any)"; fi

$(CTRL_HERE)_ref/libmlctrl.so: $(CTRL_HERE)ref/mlctrl.cpp $(INC)/mlb200.h
	mkdir -p $(CTRL_HERE)_ref
	$(CXX) $(REF_FLAGS) -O2 -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(E2S_SRC) -lpthread

.PHONY: ctrl-port ctrl-ref
