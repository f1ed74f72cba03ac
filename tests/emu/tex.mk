# TEST INFRASTRUCTURE — builds the host emulation of the texture twins of the RGBA16F and R11G11B10F kernels (emu_tex.cpp; see
# include/cuda_emu.h).  Written under a temporary name and renamed: parallel test workers may build it at the same time and must never
# load a partial file.
CXX ?= g++
CSRC = ../../fidelityfx-fsr_b200/csrc
libfsr1_emu_tex.so: emu_tex.cpp emu_srtm_in.cpp emu_post.cpp include/cuda_emu.h include/fsr1_emu_ptx.h include/fsr1_emu_surf.h \
                    include/fsr1_emu_tex.h $(CSRC)/fsr1_easu_tiled.cu $(CSRC)/fsr1_rcas_packed.cu $(CSRC)/fsr1_fused.cu \
                    $(CSRC)/fsr1_easu_quad.cuh $(CSRC)/fsr1_rcas_math.cuh $(CSRC)/fsr1_post.cuh $(CSRC)/fsr1_r11.cuh \
                    $(CSRC)/fsr1_easu_common.cuh $(CSRC)/fsr1_common.cuh
	$(CXX) -std=c++17 -O1 -fPIC -shared -pthread -x c++ -DFSR1_CPU_EMU -ffp-contract=off -w -Wl,-Bsymbolic -I include -o $@.$$$$ emu_tex.cpp && mv -f $@.$$$$ $@
