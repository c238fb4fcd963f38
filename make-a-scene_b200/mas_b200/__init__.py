"""Host side of the H100-native VQ-IMG hot path: ctypes binding (_lib), autograd units (ops), builder (build)."""
from . import _lib  # noqa: F401
from ._lib import IMPL_AUTO, IMPL_SIMT, IMPL_TC, launch_count  # noqa: F401
