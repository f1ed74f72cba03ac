# TEST INFRASTRUCTURE — builds the host emulation of fsr1_rcas_post's input-stage RCAS kernels (emu_rcas_in.cpp; see include/cuda_emu.h).
# Written under a temporary name and renamed: parallel test workers may build it at the same time and must never load a partial file.
CXX ?= g++
CSRC = ../../fidelityfx-fsr_b200/csrc
libfsr1_emu_rcas_in.so: emu_rcas_in.cpp emu_post.cpp include/cuda_emu.h include/fsr1_emu_ptx.h include/fsr1_emu_surf.h \
                        $(CSRC)/fsr1_easu_tiled.cu $(CSRC)/fsr1_rcas_packed.cu $(CSRC)/fsr1_rcas_in.cu $(CSRC)/fsr1_fused.cu $(CSRC)/fsr1_easu_quad.cuh \
                        $(CSRC)/fsr1_rcas_math.cuh $(CSRC)/fsr1_post.cuh $(CSRC)/fsr1_r11.cuh $(CSRC)/fsr1_easu_common.cuh $(CSRC)/fsr1_common.cuh
	$(CXX) -std=c++17 -O1 -fPIC -shared -pthread -x c++ -DFSR1_CPU_EMU -ffp-contract=off -w -Wl,-Bsymbolic -I include -o $@.$$$$ emu_rcas_in.cpp && mv -f $@.$$$$ $@
