"""PCIe both directions at once: copy engines vs SM-driven copies of mapped pinned memory, per CTA count."""
import sys, os, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import elodin_b200 as el
from elodin_b200 import _lib
L = _lib.lib()
h2d, d2h = 160 << 20, 104 << 20
buf = el.pinned_empty((h2d + d2h) // 8, np.float64, device=0); buf[...] = 1.0
out = (C.c_double * 2)()
_lib.check(L.b200_probe_pcie_gbs(0, C.c_void_p(buf.ctypes.data), h2d, d2h, 5, out)); print("copy engines       H2D %.1f  D2H %.1f GB/s" % (out[0], out[1]))
for blocks in (16, 32, 64, 132, 264, 528):
    _lib.check(L.b200_probe_zero_copy_gbs(0, C.c_void_p(buf.ctypes.data), h2d, d2h, 5, blocks, out)); print("kernels, %3d CTAs   H2D %.1f  D2H %.1f GB/s" % (blocks, out[0], out[1]))
for blocks in (64, 132):
    _lib.check(L.b200_probe_zero_copy_gbs(0, C.c_void_p(buf.ctypes.data), h2d, 0, 5, blocks, out)); print("kernels, %3d CTAs   H2D alone %.1f GB/s" % (blocks, out[0]))
    _lib.check(L.b200_probe_zero_copy_gbs(0, C.c_void_p(buf.ctypes.data), 0, d2h, 5, blocks, out)); print("kernels, %3d CTAs   D2H alone %.1f GB/s" % (blocks, out[1]))
_lib.check(L.b200_probe_pcie_gbs(0, C.c_void_p(buf.ctypes.data), h2d, 0, 5, out)); print("copy engine H2D alone %.1f GB/s" % out[0])
