"""Device plumbing: contexts, device arrays (torch tensors as the allocator) and streams.

PyTorch is used for device memory, streams and torch.distributed only; every computation on
the hot path goes through the C ABI (elfi_b200._lib).
"""
import ctypes

import numpy as np
import torch

from . import _lib

_contexts = {}


def require_cuda():
    if not torch.cuda.is_available():
        raise _lib.ElfiB200Error(
            "elfi_b200 needs a CUDA device (H100, sm_90a); none is visible and there is no "
            "CPU fallback.")


def current_device():
    require_cuda()
    return torch.cuda.current_device()


def context(device=None):
    """Return the (cached) elfi_b200 context handle of a device ordinal."""
    if device is None:
        device = current_device()
    if isinstance(device, torch.device):
        device = device.index if device.index is not None else torch.cuda.current_device()
    ctx = _contexts.get(device)
    if ctx is None:
        require_cuda()
        handle = ctypes.c_void_p()
        _lib.call('elfi_b200_ctx_create', int(device), ctypes.byref(handle))
        ctx = handle
        _contexts[device] = ctx
        torch.cuda.set_device(device)
    return ctx


def destroy_contexts():
    for dev, ctx in list(_contexts.items()):
        _lib.call('elfi_b200_ctx_destroy', ctx)
        del _contexts[dev]


def gpu_numa_node(device=None):
    """NUMA node the GPU's PCIe root hangs off (sysfs), or None when it cannot be determined."""
    require_cuda()
    device = torch.cuda.current_device() if device is None else int(device)
    props = torch.cuda.get_device_properties(device)
    try:
        addr = '{:04x}:{:02x}:{:02x}.0'.format(props.pci_domain_id, props.pci_bus_id,
                                               props.pci_device_id)
        with open('/sys/bus/pci/devices/{}/numa_node'.format(addr)) as f:
            node = int(f.read().strip())
        return node if node >= 0 else None
    except (OSError, AttributeError, ValueError):
        return None


def bind_to_gpu_numa_node(device=None):
    """Run this process on the cores of the GPU's NUMA node, so that the pinned staging buffers
    it allocates afterwards (first touch) are local to the GPU's PCIe root: with 8 ranks on a
    two-socket host, H2D copies from the remote socket cross the inter-socket link and slow down.
    Returns the node (None: nothing was changed).  Call before allocating host buffers."""
    import os
    node = gpu_numa_node(device)
    if node is None or not hasattr(os, 'sched_setaffinity'):
        return None
    try:
        with open('/sys/devices/system/node/node{}/cpulist'.format(node)) as f:
            spec = f.read().strip()
        cpus = set()
        for part in spec.split(','):
            lo, _, hi = part.partition('-')
            cpus.update(range(int(lo), int(hi or lo) + 1))
        cpus &= os.sched_getaffinity(0)
        if cpus:
            os.sched_setaffinity(0, cpus)
            return node
    except (OSError, ValueError):
        pass
    return None


def pinned_empty(shape, dtype=np.float64):
    """Page-locked host array (numpy view of a pinned torch tensor): H2D / D2H copies of it run
    at the PCIe rate without a staging copy."""
    tdtype = {np.float64: torch.float64, np.float32: torch.float32, np.int32: torch.int32,
              np.int64: torch.int64}[np.dtype(dtype).type]
    return torch.empty(shape, dtype=tdtype).pin_memory().numpy()


def stream_ptr():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def synchronize():
    """Wait for the work queued on the current stream."""
    require_cuda()
    torch.cuda.current_stream().synchronize()


def is_device_array(x):
    return isinstance(x, torch.Tensor) and x.is_cuda


def to_device(x, dtype=torch.float64):
    """numpy / sequence / tensor -> contiguous CUDA tensor of `dtype` on the current device."""
    require_cuda()
    if isinstance(x, torch.Tensor):
        t = x
        if not t.is_cuda:
            t = t.cuda()
        if t.dtype != dtype:
            t = t.to(dtype)
        return t.contiguous()
    arr = np.ascontiguousarray(x, dtype=_np_dtype(dtype))
    return torch.from_numpy(arr).cuda()


def to_host(x):
    """CUDA tensor -> numpy array (a synchronising copy); numpy passes through."""
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    return np.asarray(x)


def empty(shape, dtype=torch.float64):
    require_cuda()
    return torch.empty(shape, dtype=dtype, device='cuda')


def zeros(shape, dtype=torch.float64):
    require_cuda()
    return torch.zeros(shape, dtype=dtype, device='cuda')


def ones(shape, dtype=torch.float64):
    require_cuda()
    return torch.ones(shape, dtype=dtype, device='cuda')


def full(shape, value, dtype=torch.float64):
    require_cuda()
    return torch.full(shape, value, dtype=dtype, device='cuda')


def ptr(t):
    """Device (or host) pointer of a tensor / numpy array as c_void_p; None -> NULL."""
    if t is None:
        return ctypes.c_void_p(0)
    if isinstance(t, torch.Tensor):
        return ctypes.c_void_p(t.data_ptr())
    return ctypes.c_void_p(t.ctypes.data)


def _np_dtype(dtype):
    return {torch.float64: np.float64, torch.float32: np.float32, torch.int32: np.int32,
            torch.int64: np.int64, torch.uint32: np.uint32}[dtype]
