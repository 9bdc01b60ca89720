"""CUDA-tensor arguments of the query methods (TriangleMeshDistance.signed_distance / unsigned_distance,
CubicLagrangeDiscreteGrid.interpolate): which arguments take the device route, and the checks they pass before their
pointers reach a _device entry point of the C-ABI."""
import sys

from . import _capi as capi


def is_device_query(x):
    """True for a torch tensor on a CUDA device.  Under the CPU-emulated test build, whose "device" memory is host memory, every torch
    tensor takes the device route, so that the test rehearsal exercises it."""
    torch = sys.modules.get("torch")          # a caller that passes a tensor has imported torch
    if torch is None or not isinstance(x, torch.Tensor):
        return False
    return capi.EMULATED or x.is_cuda


def points(x, device, who):
    """x as a contiguous float64 (n, 3) tensor on `device` (the CUDA device of the handle it is queried against).  The results are the
    reference's fp64 bits, so another dtype is refused rather than converted."""
    import torch
    if x.dtype != torch.float64:
        raise TypeError(f"{who}: points must be a float64 tensor (got {x.dtype}); convert with x.double()")
    if not capi.EMULATED and x.device.index != device:
        raise ValueError(f"{who}: points are on {x.device} but the handle lives on cuda:{device}")
    if x.shape[-1:] != (3,) or x.dim() not in (1, 2):
        raise ValueError(f"{who}: points must have shape (n, 3) or (3,), got {tuple(x.shape)}")
    return x.reshape(-1, 3).contiguous()


def stream(x):
    """the cudaStream_t of torch's current stream on x's device (NULL under the emulated build)"""
    if capi.EMULATED:
        return None
    import torch
    return torch.cuda.current_stream(x.device).cuda_stream
