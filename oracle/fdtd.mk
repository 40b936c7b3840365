# oracle/fdtd.mk -- builds the two CPU checkers of kernel K9 (TEST INFRASTRUCTURE ONLY), with the flags of
# oracle/Makefile (included for REF, REF_FLAGS, PORT_FLAGS and E2S_SRC):
#
#   _port/libmlport_fdtd.so  plain-C restatement of the FDTD membrane (oracle/port/mlport_fdtd.c), anywhere
#   _ref/libmlfdtd.so        the reference's examples/audio-and-midi/fdtd.cpp itself: its text, extracted byte for
#                            byte into the git-ignored tests/cpp/_ref/fdtd_body.inc by tests/cpp/make_fdtd_body.py,
#                            included by oracle/ref/mlfdtd.cpp and linked with the reference's MLAudioContext.cpp
#                            and the EventsToSignals sources it needs.  Only where the reference tree and the
#                            extracted text exist; the built .so travels with the other oracle/_ref libraries.
#
#   make -f oracle/fdtd.mk fdtd-port | fdtd-ref
FDTD_HERE := $(dir $(abspath $(lastword $(MAKEFILE_LIST))))
include $(FDTD_HERE)Makefile
FDTD_BODY := $(FDTD_HERE)../tests/cpp/_ref/fdtd_body.inc

fdtd-port: $(FDTD_HERE)_port/libmlport_fdtd.so

$(FDTD_HERE)_port/libmlport_fdtd.so: $(FDTD_HERE)port/mlport_fdtd.c $(INC)/mlb200.h
	mkdir -p $(FDTD_HERE)_port
	$(CC) $(PORT_FLAGS) -o $@ $< -lm

fdtd-ref:
	@if [ -d "$(REF)/source/DSP" ] && [ -f "$(FDTD_BODY)" ]; then \
	  $(MAKE) -f $(FDTD_HERE)fdtd.mk $(FDTD_HERE)_ref/libmlfdtd.so; \
	else echo "reference tree or extracted fdtd.cpp text not present: keeping prebuilt oracle/_ref (if any)"; fi

$(FDTD_HERE)_ref/libmlfdtd.so: $(FDTD_HERE)ref/mlfdtd.cpp $(FDTD_BODY)
	mkdir -p $(FDTD_HERE)_ref
	$(CXX) $(REF_FLAGS) -include mutex -include cstring -I$(REF)/source/matrix -I$(REF)/external/utf \
	  -o $@ $< $(REF)/source/app/MLAudioContext.cpp $(E2S_SRC) -lpthread

.PHONY: fdtd-port fdtd-ref
