"""FSR_Filter — host-side mirror of the reference's filter object (the operator boundary).

Reference: sample/src/DX12/FSR_Filter.h:27-45 and FSR_Filter.cpp:41-141 (VK twin sample/src/VK/FSR_Filter.cpp).
Same method names, argument meaning and call pattern; D3D12 objects are replaced by torch CUDA tensors
(device memory) and a CUDA stream (the command list).  The C++ twin for native callers is
fsr_filter.hpp (same directory).
"""
from dataclasses import dataclass

import torch

from . import api

UPSCALE_TYPE_BILINEAR = 0  # the sample's comparison mode (FSR_Pass.hlsl:70-73) is out of scope: rejected
UPSCALE_TYPE_FSR_1_0 = 1

# quality presets of the sample (sample/src/DX12/FSRSample.h:70-97): display / ratio, truncating
PRESETS = {"ultra_quality": 1.3, "quality": 1.5, "balanced": 1.7, "performance": 2.0}


def render_resolution(display_w, display_h, ratio):
    return int(display_w / ratio), int(display_h / ratio)


@dataclass
class State:
    """The fields of the sample's State that Upscale reads (sample/src/DX12/SampleRenderer.h:36-60)."""
    renderWidth: int = 0
    renderHeight: int = 0
    bUseRcas: bool = True
    rcasAttenuation: float = 0.25
    m_nUpscaleType: int = UPSCALE_TYPE_FSR_1_0


class FSR_Filter:
    def __init__(self):
        self._device = None
        self._intermediary = None
        self._display = None
        self._dtype = None
        self.flags = 0

    def OnCreate(self, device=None, dtype=torch.float16, slowFallback=False):
        """FSR_Filter::OnCreate (FSR_Filter.cpp:41-68): pick the fp16 or the fp32 ("slow fallback") kernels."""
        if not torch.cuda.is_available():
            raise api.Fsr1Error("FSR_Filter needs a CUDA device; there is no CPU path")
        self._device = torch.device(device if device is not None else "cuda")
        self._dtype = torch.float32 if slowFallback else dtype
        api._lib.lib()  # fail now, loudly, if the CUDA library is missing

    def OnCreateWindowSizeDependentResources(self, renderWidth, renderHeight, displayWidth, displayHeight):
        """FSR_Filter::OnCreateWindowSizeDependentResources (FSR_Filter.cpp:70-90): the display-sized intermediate."""
        self._display = (int(displayWidth), int(displayHeight))
        self._render = (int(renderWidth), int(renderHeight))
        self._intermediary = torch.empty((displayHeight, displayWidth, 4), dtype=self._dtype, device=self._device)

    def OnDestroyWindowSizeDependentResources(self):
        self._intermediary = None

    def OnDestroy(self):
        self.OnDestroyWindowSizeDependentResources()
        self._device = None

    def Upscale(self, inputTexture, outputTexture, displayWidth, displayHeight, pState, stream=None, hdr=False):
        """FSR_Filter::Upscale (FSR_Filter.cpp:101-141): constants, EASU dispatch, RCAS dispatch."""
        if pState.m_nUpscaleType != UPSCALE_TYPE_FSR_1_0:
            raise api.Fsr1Error("only the FSR 1.0 path is implemented (bilinear comparison mode is out of scope)")
        # hdr: the sample's Sample.x == 1 (FSR_Filter.cpp:107,125: `hdr && !bUseRcas` for EASU, `hdr` for RCAS):
        # the LAST pass squares its output (gamma 2.0 from TEPD back to linear)
        flags = self.flags | (api.FLAG_OUTPUT_SQUARE if hdr else 0)
        if self._intermediary is None or self._display != (displayWidth, displayHeight):
            raise api.Fsr1Error("call OnCreateWindowSizeDependentResources for this display size first")
        rw, rh = int(pState.renderWidth), int(pState.renderHeight)
        if rw <= 0 or rh <= 0 or rw > inputTexture.shape[1] or rh > inputTexture.shape[0]:
            raise api.Fsr1Error("render size %dx%d does not fit the %dx%d input texture"
                                % (rw, rh, inputTexture.shape[1], inputTexture.shape[0]))
        # the constants describe an input of exactly the render size: taps clamp at the render region's edge, so only that
        # region is described (as fsr_filter.hpp does through fsr1_context_upscale_render)
        inputTexture = inputTexture[:rh, :rw]
        econ = api.easu_con(rw, rh, rw, rh, displayWidth, displayHeight)
        if pState.bUseRcas:
            rcon = api.rcas_con(pState.rcasAttenuation)
            api.upscale(inputTexture, self._intermediary, outputTexture, econ, rcon, flags=flags, stream=stream)
        else:
            api.easu(inputTexture, outputTexture, econ, flags=flags, stream=stream)
        return outputTexture
