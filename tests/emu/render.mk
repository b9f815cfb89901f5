# CPU build of the camera-image device code (test infrastructure only): make -C tests/emu -f render.mk OUT=<dir>
# OUT defaults to _build; the tests pass a temporary directory so that the source tree may be read-only.
CXX ?= g++
CXXFLAGS ?= -O2 -fPIC -std=c++17 -x c++ -Wall -Wno-unknown-pragmas -Wno-unused-variable -ffp-contract=off
OUT ?= _build
all: $(OUT)/libb2q_emu_render.so
$(OUT)/libb2q_emu_render.so: emu_render.cpp ../../paddlerobotics_b200/csrc/b2q_render.cuh ../../paddlerobotics_b200/csrc/b2q_sim.cuh ../../paddlerobotics_b200/csrc/b2q_math.cuh ../../paddlerobotics_b200/csrc/b2q_model_host.h
	mkdir -p $(OUT)
	$(CXX) $(CXXFLAGS) -shared -o $@ emu_render.cpp
