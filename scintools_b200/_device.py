"""Device plumbing: torch is used for device buffers, streams and
torch.distributed only.  All arithmetic is in libscint_b200."""
import os

import numpy as np

from . import _lib

_state = {"dev": None}


def device():
    """Initialise (once) and return the torch device of this process."""
    if _state["dev"] is None:
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError(
                "scintools_b200 needs a CUDA (sm_90a) device; there is no "
                "CPU fallback")
        idx = int(os.environ.get("LOCAL_RANK", "0")) % torch.cuda.device_count()
        torch.cuda.set_device(idx)
        _lib.check(_lib.lib.sb_init(idx))
        _state["dev"] = torch.device("cuda", idx)
    return _state["dev"]


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def ptr(t):
    return 0 if t is None else t.data_ptr()


def empty(shape, dtype):
    import torch
    return torch.empty(shape, dtype=dtype, device=device())


def zeros(shape, dtype):
    import torch
    return torch.zeros(shape, dtype=dtype, device=device())


def upload(arr, pin=False):
    """numpy -> device tensor, same dtype (complex -> trailing dim of 2)."""
    import torch
    dev = device()
    a = np.ascontiguousarray(arr)
    if np.iscomplexobj(a):
        a = a.view(a.real.dtype).reshape(a.shape + (2,))
    t = torch.from_numpy(a)
    if pin:
        t = t.pin_memory()
    return t.to(dev, non_blocking=pin)


def upload_f32(arr, pin=False):
    """numpy (real or complex, any float width) -> float32 device tensor.
    float64 input is uploaded unchanged and narrowed on the device by
    sb_convert_f64_f32, so the host never makes a pass over the data."""
    import torch
    a = np.asarray(arr)
    if a.dtype not in (np.float32, np.float64, np.complex64, np.complex128):
        a = a.astype(np.complex128 if np.iscomplexobj(a) else np.float64)
    t = upload(a, pin)
    if t.dtype == torch.float32:
        return t
    out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
    _lib.check(_lib.lib.sb_convert_f64_f32(t.data_ptr(), out.data_ptr(),
                                           t.numel(), stream_ptr()))
    return out


def download(t, dtype=None):
    a = t.cpu().numpy()
    if dtype is not None and a.dtype != dtype:
        a = a.astype(dtype)
    return a
