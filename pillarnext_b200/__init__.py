"""pillarnext_b200 -- H100 (sm_90a) native hot path of PillarNeXt-B behind the reference's det3d module API.

csrc/ + libpnx.so : hand-written CUDA kernels behind the C-ABI in include/pnx.h
ops.py            : device-buffer plumbing (torch) -> C-ABI calls
functional.py     : autograd.Functions (forward + backward in libpnx)
modules.py        : nn.Module mirror of the reference classes (same names / kwargs / state-dict keys)
synth.py          : synthetic nuScenes-/Waymo-shaped inputs
"""
__version__ = "0.1.0"
