"""Helpers for the -m gpu parity tests: raw device buffers through the C ABI."""
import ctypes as C

import numpy as np

from stencil_b200._lib import Pitched, check, lib


class DevArray:
    """A 3-D [z,y,x] array in device memory (unpitched, like the reference's allocations)."""

    def __init__(self, host: np.ndarray, device: int = 0, extra: int = 0, lead: int = 0):
        """lead: bytes between the start of the sb_malloc block (256-byte aligned) and element 0, as LocalDomain leaves
        in front of an allocation so that its first compute cell is 16-byte aligned."""
        host = np.ascontiguousarray(host)
        self.shape, self.dtype, self.device = host.shape, host.dtype, device
        self.nbytes = host.nbytes
        p = C.c_void_p()
        check(lib().sb_malloc(C.byref(p), max(lead + self.nbytes + extra, 16), device))
        self.base = int(p.value)
        self.ptr = self.base + lead
        check(lib().sb_memcpy(C.c_void_p(self.ptr), host.ctypes.data, self.nbytes, device, None))
        check(lib().sb_stream_sync(device, None))

    def pitched(self) -> Pitched:
        assert len(self.shape) == 3
        return Pitched(self.ptr, self.shape[2] * self.dtype.itemsize, self.shape[1])

    def get(self) -> np.ndarray:
        out = np.empty(self.shape, dtype=self.dtype)
        check(lib().sb_device_sync(self.device))
        check(lib().sb_memcpy(out.ctypes.data, C.c_void_p(self.ptr), self.nbytes, self.device, None))
        check(lib().sb_stream_sync(self.device, None))
        return out

    def free(self):
        if self.ptr:
            lib().sb_free(C.c_void_p(self.base), self.device)
            self.ptr = 0

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def oracle_radius(r):
    """stencil_b200.Radius -> oracle.geometry.Radius"""
    from oracle import geometry as g

    out = g.Radius()
    for z in (-1, 0, 1):
        for y in (-1, 0, 1):
            for x in (-1, 0, 1):
                out.set_dir((x, y, z), r.dir((x, y, z)))
    return out
