"""zetaray_b200 -- H100-native ReSTIR path-tracing core behind ZetaRay's render-pass interface.

The product is `libzetaray_b200.so` (hand-written sm_90a CUDA behind the C-ABI of include/zr_abi.h).
This package is the thin Python binding used by the tests and bench.py: ctypes prototypes plus
host-side mirrors of the reference's pass objects (zetaray_b200.passes). There is no CPU fallback:
importing `lib` fails loudly if the shared library has not been built."""
from . import _lib  # noqa: F401
from ._lib import lib, check, ZRError  # noqa: F401
