"""Compile the reference's own rotated-NMS CUDA extension (det3d/core/iou3d_nms/src/{iou3d_nms_api.cpp, iou3d_nms.cpp,
iou3d_nms_kernel.cu, iou3d_cpu.cpp}) for sm_90a into oracle/_ref/ref_iou3d_nms.so (TEST INFRASTRUCTURE).  Sources are
compiled where they lie under the reference tree (nothing is copied); the recipe is torch.utils.cpp_extension (nvcc +
g++ + ninja) with the reference setup.py's nvcc optimisation level, not its setup.py.  The module exposes the reference's
`nms_gpu(boxes, keep, thr)` and `boxes_iou_bev_gpu(a, b, out)`: the GPU NMS the reference's predict runs
(rotate_nms_pcdet), the oracle of tests/test_production_postproc_gpu.py."""
import os
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(os.environ.get("PNX_REFERENCE_ROOT", "/root/reference"), "det3d/core/iou3d_nms/src")
SOURCES = ["iou3d_nms_api.cpp", "iou3d_nms.cpp", "iou3d_nms_kernel.cu", "iou3d_cpu.cpp"]
OUT = os.path.join(ROOT, "_ref")
NAME = "ref_iou3d_nms"
SO = os.path.join(OUT, NAME + ".so")


def available():
    return all(os.path.isfile(os.path.join(REF_DIR, s)) for s in SOURCES)


def _import(so):
    import importlib.util
    import torch  # noqa: F401  (libtorch must be loaded first)
    spec = importlib.util.spec_from_file_location(NAME, so)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def load(build=True):
    """Returns the extension module or None.  build=False only imports a prebuilt oracle/_ref/ref_iou3d_nms.so and never
    looks at the reference tree (which machines that only run the tests do not have)."""
    if not build:
        return _import(SO) if os.path.isfile(SO) else None
    srcs = [os.path.join(REF_DIR, s) for s in SOURCES]
    if os.path.isfile(SO) and (not available() or os.path.getmtime(SO) >= max(os.path.getmtime(s) for s in srcs)):
        return _import(SO)
    if not available():
        return None
    from torch.utils.cpp_extension import load as cpp_load
    os.makedirs(OUT, exist_ok=True)
    prev = os.environ.get("TORCH_CUDA_ARCH_LIST")
    os.environ["TORCH_CUDA_ARCH_LIST"] = "9.0a"
    try:
        cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
        return cpp_load(name=NAME, sources=srcs, build_directory=OUT, extra_include_paths=[cuda_inc, REF_DIR],
                        extra_cflags=["-O2", "-w"], extra_cuda_cflags=["-O2", "-w"], verbose=False)
    finally:
        if prev is None:
            os.environ.pop("TORCH_CUDA_ARCH_LIST", None)
        else:
            os.environ["TORCH_CUDA_ARCH_LIST"] = prev


if __name__ == "__main__":
    m = load()
    print("built" if m is not None else "reference source not present", file=sys.stderr)
