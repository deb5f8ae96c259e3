"""rustfft_b200 -- H100-native batched complex FFT behind RustFFT's FftPlanner / Fft interface.

Host-side mirror (Python, because the image has no Rust toolchain) of the reference's public
API for the hot path; the names, argument meaning and error behaviour follow the reference
(paths relative to the RustFFT 6.4.1 tree):

    FftPlanner.plan_fft / plan_fft_forward / plan_fft_inverse      src/plan.rs:67-126
    Fft.process / process_with_scratch                             src/lib.rs:195-211
    Fft.process_outofplace_with_scratch                            src/lib.rs:231-236
    Fft.process_immutable_with_scratch                             src/lib.rs:250-255
    Fft.get_{inplace,outofplace,immutable}_scratch_len             src/lib.rs:262-277
    Fft.len / Fft.fft_direction                                    src/lib.rs:140-181
    FftDirection                                                   src/lib.rs:147-171

Everything numeric happens in rustfft_b200/libb200fft.so (hand-written sm_90a CUDA behind the
C ABI of include/b200fft.h).  There is no CPU fallback: without the library or without an H100
the planner raises.  PyTorch is only used for device memory / streams by callers (tests, bench).
"""
from __future__ import annotations

import ctypes
import enum
import os
import re
import threading
from typing import Dict, Optional, Tuple

import numpy as np

__all__ = ["FftDirection", "FftPlanner", "Fft", "Library", "FftError", "Recipe", "RealFftPlanner", "RealFft", "RealFft2d", "Fft2d", "FftConvolution",
           "ChannelConvolution", "FftConvolution2d", "DctKind", "DctPlanner", "Dct", "DctNd", "Stft", "Czt", "Hilbert", "Mdct", "mdct_window",
           "default_library", "shard_range"]

_HERE = os.path.dirname(os.path.abspath(__file__))
# B200FFT_LIB: load another build of the same C ABI (A/B measurements of kernel variants; tools/ab_two_pass.py)
DEFAULT_LIB_PATH = os.environ.get("B200FFT_LIB") or os.path.join(_HERE, "libb200fft.so")

F32, F64 = 0, 1


class FftError(RuntimeError):
    """Raised where the reference panics (src/common.rs:13-104) or where CUDA fails."""

    def __init__(self, code: int, message: str):
        super().__init__(message)
        self.code = code


class FftDirection(enum.IntEnum):
    Forward = 0
    Inverse = 1

    def opposite_direction(self) -> "FftDirection":  # src/lib.rs:156-161
        return FftDirection.Inverse if self == FftDirection.Forward else FftDirection.Forward


class _RecipeNode(ctypes.Structure):  # b200fft_recipe_node (include/b200fft.h)
    _fields_ = [("kind", ctypes.c_uint32), ("child", ctypes.c_uint32), ("len", ctypes.c_uint64), ("a", ctypes.c_uint64), ("b", ctypes.c_uint64)]


class Recipe:
    """A decomposition chosen by the host (the reference's Recipe enum, src/plan.rs:134-226) handed to the library as data.

    Built with the class methods; `inner` is the Recipe of the inner FFT of a Rader / Bluestein node."""

    AUTO, POW2, SMOOTH, MIXED_RADIX, GOOD_THOMAS, RADER, BLUESTEIN, CLUSTER = range(8)

    def __init__(self, kind: int, len: int, a: int = 0, b: int = 0, inner: Optional["Recipe"] = None):
        self.kind, self.len, self.a, self.b, self.inner = kind, int(len), int(a), int(b), inner

    @classmethod
    def pow2(cls, n):
        return cls(cls.POW2, n)

    @classmethod
    def cluster(cls, n, half_tiles=False):
        return cls(cls.CLUSTER, n, 1 if half_tiles else 0)

    def to_dict(self):
        """JSON-friendly form (plan serialisation): Recipe.from_dict(json.loads(json.dumps(r.to_dict()))) rebuilds the same plan."""
        d = {"kind": self.kind, "len": self.len, "a": self.a, "b": self.b}
        if self.inner is not None:
            d["inner"] = self.inner.to_dict()
        return d

    @classmethod
    def from_dict(cls, d):
        return cls(d["kind"], d["len"], d.get("a", 0), d.get("b", 0), cls.from_dict(d["inner"]) if d.get("inner") else None)

    @classmethod
    def smooth(cls, n):
        return cls(cls.SMOOTH, n)

    @classmethod
    def mixed_radix(cls, a, b):
        return cls(cls.MIXED_RADIX, a * b, a, b)

    @classmethod
    def good_thomas(cls, a, b):
        return cls(cls.GOOD_THOMAS, a * b, a, b)

    @classmethod
    def rader(cls, n, outer_radix=1, inner: Optional["Recipe"] = None):
        return cls(cls.RADER, n, outer_radix, 0, inner)

    @classmethod
    def bluestein(cls, n, inner: Optional["Recipe"] = None):
        return cls(cls.BLUESTEIN, n, 0, 0, inner)

    def flatten(self):
        nodes, r = [], self
        while r is not None:
            nodes.append(r)
            r = r.inner
        arr = (_RecipeNode * len(nodes))()
        for i, r in enumerate(nodes):
            arr[i] = _RecipeNode(r.kind, i + 1 if r.inner is not None else 0, r.len, r.a, r.b)
        return arr


class Library:
    """A loaded C-ABI library (include/b200fft.h)."""

    SYMBOLS = [
        "b200fft_device_count", "b200fft_plan_create", "b200fft_plan_create_from_recipe", "b200fft_plan_recipe", "b200fft_plan_destroy",
        "b200fft_plan_len",
        "b200fft_plan_direction", "b200fft_plan_precision", "b200fft_plan_scratch_len", "b200fft_plan_describe",
        "b200fft_plan_launches", "b200fft_exec_host_inplace", "b200fft_exec_host_outofplace", "b200fft_exec_device",
        "b200fft_workspace_bytes", "b200fft_exec_device_ws", "b200fft_last_error", "b200fft_version",
        "b200fft_real_plan_create", "b200fft_real_plan_destroy", "b200fft_real_workspace_bytes", "b200fft_real_forward_device",
        "b200fft_real_inverse_device", "b200fft_real_forward_host", "b200fft_real_inverse_host",
        "b200fft_plan2d_create", "b200fft_plan2d_destroy", "b200fft_exec2d_device", "b200fft_exec2d_host",
        "b200fft_conv_plan_create", "b200fft_conv_plan_destroy", "b200fft_conv_output_len", "b200fft_conv_describe",
        "b200fft_conv_device", "b200fft_conv_host",
        "b200fft_chconv_plan_create", "b200fft_chconv_plan_destroy", "b200fft_chconv_output_len", "b200fft_chconv_describe",
        "b200fft_chconv_device", "b200fft_chconv_host",
        "b200fft_real_plan2d_create", "b200fft_real_plan2d_destroy", "b200fft_real_plan2d_describe", "b200fft_real2d_forward_device",
        "b200fft_real2d_inverse_device", "b200fft_real2d_forward_host", "b200fft_real2d_inverse_host",
        "b200fft_conv2d_plan_create", "b200fft_conv2d_plan_destroy", "b200fft_conv2d_output_shape", "b200fft_conv2d_describe",
        "b200fft_conv2d_device", "b200fft_conv2d_host",
        "b200fft_dct_plan_create", "b200fft_dct_plan_destroy", "b200fft_dct_describe", "b200fft_dct_device", "b200fft_dct_host",
        "b200fft_dctn_plan_create", "b200fft_dctn_plan_destroy", "b200fft_dctn_describe", "b200fft_dctn_device", "b200fft_dctn_host",
        "b200fft_stft_plan_create", "b200fft_stft_plan_destroy", "b200fft_stft_describe", "b200fft_stft_frames",
        "b200fft_stft_forward_device", "b200fft_stft_inverse_device", "b200fft_stft_forward_host", "b200fft_stft_inverse_host",
        "b200fft_czt_plan_create", "b200fft_czt_plan_destroy", "b200fft_czt_describe", "b200fft_czt_device", "b200fft_czt_host",
        "b200fft_hilbert_plan_create", "b200fft_hilbert_plan_destroy", "b200fft_hilbert_describe", "b200fft_hilbert_device",
        "b200fft_hilbert_host",
        "b200fft_mdct_plan_create", "b200fft_mdct_plan_destroy", "b200fft_mdct_describe", "b200fft_mdct_frames",
        "b200fft_mdct_forward_device", "b200fft_mdct_inverse_device", "b200fft_mdct_forward_host", "b200fft_mdct_inverse_host",
        "b200fft_plan3d_create", "b200fft_plan3d_destroy", "b200fft_plan3d_describe", "b200fft_exec3d_device", "b200fft_exec3d_host",
        "b200fft_real_plan3d_create", "b200fft_real_plan3d_destroy", "b200fft_real_plan3d_describe", "b200fft_real3d_forward_device",
        "b200fft_real3d_inverse_device", "b200fft_real3d_forward_host", "b200fft_real3d_inverse_host",
    ]

    def __init__(self, path: str = DEFAULT_LIB_PATH):
        if not os.path.exists(path):
            raise FftError(-2, f"{path} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback)")
        self.path = path
        self.c = ctypes.CDLL(path)
        c, u64, i32, vp = self.c, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p
        c.b200fft_device_count.argtypes = [ctypes.POINTER(i32)]
        c.b200fft_plan_create.argtypes = [ctypes.POINTER(vp), u64, i32, i32, i32]
        c.b200fft_plan_create_from_recipe.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(_RecipeNode), ctypes.c_uint32, i32, i32, i32]
        c.b200fft_plan_recipe.argtypes = [vp, ctypes.POINTER(_RecipeNode), ctypes.c_uint32]
        c.b200fft_plan_destroy.argtypes = [vp]
        c.b200fft_plan_len.argtypes = [vp]
        c.b200fft_plan_len.restype = u64
        c.b200fft_plan_direction.argtypes = [vp]
        c.b200fft_plan_precision.argtypes = [vp]
        c.b200fft_plan_scratch_len.argtypes = [vp, i32]
        c.b200fft_plan_scratch_len.restype = u64
        c.b200fft_plan_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_plan_launches.argtypes = [vp, u64]
        c.b200fft_plan_launches.restype = u64
        c.b200fft_exec_host_inplace.argtypes = [vp, vp, u64]
        c.b200fft_exec_host_outofplace.argtypes = [vp, vp, vp, u64]
        c.b200fft_exec_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_workspace_bytes.argtypes = [vp, u64]
        c.b200fft_workspace_bytes.restype = u64
        c.b200fft_exec_device_ws.argtypes = [vp, vp, vp, u64, vp, vp, u64]
        c.b200fft_last_error.restype = ctypes.c_char_p
        c.b200fft_version.restype = ctypes.c_char_p
        c.b200fft_real_plan_create.argtypes = [ctypes.POINTER(vp), u64, i32, i32]
        c.b200fft_real_plan_destroy.argtypes = [vp]
        c.b200fft_real_workspace_bytes.argtypes = [vp, u64]
        c.b200fft_real_workspace_bytes.restype = u64
        c.b200fft_real_forward_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real_inverse_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real_forward_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_real_inverse_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_plan2d_create.argtypes = [ctypes.POINTER(vp), u64, u64, i32, i32, i32]
        c.b200fft_plan2d_destroy.argtypes = [vp]
        c.b200fft_exec2d_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_exec2d_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_conv_plan_create.argtypes = [ctypes.POINTER(vp), u64, vp, u64, i32, i32, i32, i32]
        c.b200fft_conv_plan_destroy.argtypes = [vp]
        c.b200fft_conv_output_len.argtypes = [vp]
        c.b200fft_conv_output_len.restype = u64
        c.b200fft_conv_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_conv_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_conv_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_chconv_plan_create.argtypes = [ctypes.POINTER(vp), u64, u64, vp, u64, i32, i32, i32, i32, i32]
        c.b200fft_chconv_plan_destroy.argtypes = [vp]
        c.b200fft_chconv_output_len.argtypes = [vp]
        c.b200fft_chconv_output_len.restype = u64
        c.b200fft_chconv_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_chconv_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_chconv_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_real_plan2d_create.argtypes = [ctypes.POINTER(vp), u64, u64, i32, i32]
        c.b200fft_real_plan2d_destroy.argtypes = [vp]
        c.b200fft_real_plan2d_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_real2d_forward_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real2d_inverse_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real2d_forward_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_real2d_inverse_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_conv2d_plan_create.argtypes = [ctypes.POINTER(vp), u64, u64, vp, u64, u64, i32, i32, i32]
        c.b200fft_conv2d_plan_destroy.argtypes = [vp]
        c.b200fft_conv2d_output_shape.argtypes = [vp, ctypes.POINTER(u64), ctypes.POINTER(u64)]
        c.b200fft_conv2d_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_conv2d_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_conv2d_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_dct_plan_create.argtypes = [ctypes.POINTER(vp), u64, i32, i32, i32]
        c.b200fft_dct_plan_destroy.argtypes = [vp]
        c.b200fft_dct_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_dct_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_dct_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_dctn_plan_create.argtypes = [ctypes.POINTER(vp), ctypes.POINTER(u64), i32, i32, i32, i32]
        c.b200fft_dctn_plan_destroy.argtypes = [vp]
        c.b200fft_dctn_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_dctn_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_dctn_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_stft_plan_create.argtypes = [ctypes.POINTER(vp), u64, vp, u64, u64, i32, i32, i32]
        c.b200fft_stft_plan_destroy.argtypes = [vp]
        c.b200fft_stft_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_stft_frames.argtypes = [vp]
        c.b200fft_stft_frames.restype = u64
        c.b200fft_stft_forward_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_stft_inverse_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_stft_forward_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_stft_inverse_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_czt_plan_create.argtypes = [ctypes.POINTER(vp), u64, u64, ctypes.c_double, ctypes.c_double, i32, i32, i32]
        c.b200fft_czt_plan_destroy.argtypes = [vp]
        c.b200fft_czt_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_czt_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_czt_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_hilbert_plan_create.argtypes = [ctypes.POINTER(vp), u64, i32, i32]
        c.b200fft_hilbert_plan_destroy.argtypes = [vp]
        c.b200fft_hilbert_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_hilbert_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_hilbert_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_mdct_plan_create.argtypes = [ctypes.POINTER(vp), u64, vp, u64, i32, i32]
        c.b200fft_mdct_plan_destroy.argtypes = [vp]
        c.b200fft_mdct_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_mdct_frames.argtypes = [vp]
        c.b200fft_mdct_frames.restype = u64
        c.b200fft_mdct_forward_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_mdct_inverse_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_mdct_forward_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_mdct_inverse_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_plan3d_create.argtypes = [ctypes.POINTER(vp), u64, u64, u64, i32, i32, i32]
        c.b200fft_plan3d_destroy.argtypes = [vp]
        c.b200fft_plan3d_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_exec3d_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_exec3d_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_real_plan3d_create.argtypes = [ctypes.POINTER(vp), u64, u64, u64, i32, i32]
        c.b200fft_real_plan3d_destroy.argtypes = [vp]
        c.b200fft_real_plan3d_describe.argtypes = [vp, ctypes.c_char_p, u64]
        c.b200fft_real3d_forward_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real3d_inverse_device.argtypes = [vp, vp, vp, u64, vp]
        c.b200fft_real3d_forward_host.argtypes = [vp, vp, vp, u64]
        c.b200fft_real3d_inverse_host.argtypes = [vp, vp, vp, u64]

    def device_count(self) -> int:
        n = ctypes.c_int(0)
        self.check(self.c.b200fft_device_count(ctypes.byref(n)))
        return n.value

    def version(self) -> str:
        return self.c.b200fft_version().decode()

    def check(self, rc: int) -> None:
        if rc != 0:
            raise FftError(rc, self.c.b200fft_last_error().decode())


_default: Optional[Library] = None
_default_lock = threading.Lock()


def default_library() -> Library:
    global _default
    with _default_lock:
        if _default is None:
            _default = Library(DEFAULT_LIB_PATH)
        return _default


_DTYPES = {np.dtype(np.complex64): F32, np.dtype(np.complex128): F64}


class Fft:
    """One planned transform: the Arc<dyn Fft<T>> of the reference (src/lib.rs:184-278).

    Immutable after construction and safe to call from many threads (examples/concurrency.rs)."""

    def __init__(self, lib: Library, length: int, direction: FftDirection, precision: int, device: int, recipe: Optional[Recipe] = None):
        self._lib = lib
        self._h = ctypes.c_void_p()
        if recipe is not None:
            nodes = recipe.flatten()
            lib.check(lib.c.b200fft_plan_create_from_recipe(ctypes.byref(self._h), nodes, len(nodes), int(direction), precision, device))
        else:
            lib.check(lib.c.b200fft_plan_create(ctypes.byref(self._h), length, int(direction), precision, device))
        self._len = length
        self._direction = FftDirection(direction)
        self._precision = precision
        self.device = device

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_plan_destroy(h)
            except Exception:
                pass

    # ---- Length / Direction ------------------------------------------------------------
    def len(self) -> int:
        return self._len

    def __len__(self) -> int:
        return self._len

    def fft_direction(self) -> FftDirection:
        return self._direction

    @property
    def dtype(self):
        return np.complex64 if self._precision == F32 else np.complex128

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_plan_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def recipe(self) -> "Recipe":
        """The decomposition this plan was built as (b200fft_plan_recipe): feed it to FftPlanner.plan_fft_with_recipe to rebuild it."""
        arr = (_RecipeNode * 8)()
        n = self._lib.c.b200fft_plan_recipe(self._h, arr, 8)
        if n < 0:
            self._lib.check(n)
        rc = None
        for i in range(n - 1, -1, -1):
            rc = Recipe(arr[i].kind, arr[i].len, arr[i].a, arr[i].b, rc if arr[i].child else None)
        return rc

    def launches(self, batch: int) -> int:
        return int(self._lib.c.b200fft_plan_launches(self._h, batch))

    # ---- scratch getters: this backend needs no caller scratch (allowed, src/lib.rs:259-261)
    def get_inplace_scratch_len(self) -> int:
        return int(self._lib.c.b200fft_plan_scratch_len(self._h, 0))

    def get_outofplace_scratch_len(self) -> int:
        return int(self._lib.c.b200fft_plan_scratch_len(self._h, 1))

    def get_immutable_scratch_len(self) -> int:
        return int(self._lib.c.b200fft_plan_scratch_len(self._h, 2))

    # ---- host-slice trait methods ------------------------------------------------------
    def _host(self, a, name: str, writable: bool) -> np.ndarray:
        if not isinstance(a, np.ndarray) or a.dtype != np.dtype(self.dtype) or a.ndim != 1 or not a.flags.c_contiguous:
            raise TypeError(f"{name} must be a contiguous 1-D numpy array of {np.dtype(self.dtype).name}")
        if writable and not a.flags.writeable:
            raise TypeError(f"{name} must be writable")
        return a

    def _check_scratch(self, scratch, need: int) -> None:
        # "Not enough scratch space was provided..." (src/common.rs:32-37); need is 0 here, so any
        # scratch (even dirty, src/test_utils.rs:131-141) is accepted and ignored.
        if scratch is not None and len(scratch) < need:
            raise FftError(-9, f"Not enough scratch space was provided. Expected scratch len >= {need}, "
                               f"got scratch len = {len(scratch)}")

    def process(self, buffer: np.ndarray) -> None:
        """In place over every contiguous chunk of len() elements (src/lib.rs:195-198)."""
        self.process_with_scratch(buffer, None)

    def process_with_scratch(self, buffer: np.ndarray, scratch=None) -> None:
        buffer = self._host(buffer, "buffer", True)
        self._check_scratch(scratch, self.get_inplace_scratch_len())
        self._lib.check(self._lib.c.b200fft_exec_host_inplace(self._h, buffer.ctypes.data, buffer.size))

    def process_outofplace_with_scratch(self, input: np.ndarray, output: np.ndarray, scratch=None) -> None:
        """input may be used as scratch by the reference (src/lib.rs:213-236); here it is left intact."""
        input = self._host(input, "input", True)
        output = self._host(output, "output", True)
        self._check_scratch(scratch, self.get_outofplace_scratch_len())
        if input.size != output.size:
            raise FftError(-6, "Provided FFT input buffer and output buffer must have the same length. "
                               f"Got input.len() = {input.size}, output.len() = {output.size}")
        self._lib.check(self._lib.c.b200fft_exec_host_outofplace(self._h, input.ctypes.data, output.ctypes.data, input.size))

    def process_immutable_with_scratch(self, input: np.ndarray, output: np.ndarray, scratch=None) -> None:
        input = self._host(input, "input", False)
        output = self._host(output, "output", True)
        self._check_scratch(scratch, self.get_immutable_scratch_len())
        if input.size != output.size:
            raise FftError(-6, "Provided FFT input buffer and output buffer must have the same length. "
                               f"Got input.len() = {input.size}, output.len() = {output.size}")
        self._lib.check(self._lib.c.b200fft_exec_host_outofplace(self._h, input.ctypes.data, output.ctypes.data, input.size))

    # ---- device-resident path (no reference equivalent; the measured one) --------------
    def workspace_bytes(self, batch: int) -> int:
        return int(self._lib.c.b200fft_workspace_bytes(self._h, batch))

    def process_device_ptr(self, d_in: int, d_out: int, batch: int, stream: int = 0,
                           workspace: int = 0, workspace_bytes: int = 0) -> None:
        """Raw pointers on the plan's device, batch*len() elements each, async on `stream`."""
        if workspace:
            rc = self._lib.c.b200fft_exec_device_ws(self._h, d_in, d_out, batch, stream, workspace, workspace_bytes)
        else:
            rc = self._lib.c.b200fft_exec_device(self._h, d_in, d_out, batch, stream)
        self._lib.check(rc)

    def process_device(self, x, out=None, workspace=None):
        """x: torch complex tensor on the plan's device holding batch*len() elements (any shape,
        contiguous).  In place when `out` is None.  Asynchronous on torch's current stream."""
        import torch

        want = torch.complex64 if self._precision == F32 else torch.complex128
        if x.dtype != want or not x.is_cuda or not x.is_contiguous():
            raise TypeError(f"process_device wants a contiguous CUDA tensor of {want}")
        if x.device.index != self.device:
            raise FftError(-1, f"tensor is on cuda:{x.device.index}, plan is on cuda:{self.device}")
        dst = x if out is None else out
        if dst.dtype != want or dst.numel() != x.numel() or not dst.is_contiguous() or dst.device != x.device:
            raise FftError(-6, "Provided FFT input buffer and output buffer must have the same length. "
                               f"Got input.len() = {x.numel()}, output.len() = {dst.numel()}")
        n = x.numel()
        if self._len == 0 or n == 0:
            return dst
        if n < self._len:  # (an empty buffer is zero chunks and validates, src/array_utils.rs:151-177)
            raise FftError(-4, f"Provided FFT buffer was too small. Expected len = {self._len}, got len = {n}")
        if n % self._len:
            raise FftError(-5, "Input FFT buffer must be a multiple of FFT length. "
                               f"Expected multiple of {self._len}, got len = {n}")
        stream = torch.cuda.current_stream(x.device).cuda_stream
        ws_ptr, ws_bytes = 0, 0
        if workspace is not None:
            ws_ptr, ws_bytes = workspace.data_ptr(), workspace.numel() * workspace.element_size()
        self.process_device_ptr(x.data_ptr(), dst.data_ptr(), n // self._len, stream, ws_ptr, ws_bytes)
        return dst


class FftPlanner:
    """FftPlanner<T> of the reference (src/plan.rs:67-126) for this backend.

    Like FftPlannerAvx::new() (src/avx/avx_planner.rs:121-164) construction fails when the hardware
    is absent -- the reference would then fall through to its next backend; here it raises, because
    this package has no other backend.  Plans are cached per (len, direction) exactly like
    FftCache (src/fft_cache.rs:5-38): planning the same transform twice returns the same object."""

    def __init__(self, dtype=np.complex64, device: int = 0, lib: Optional[Library] = None):
        dt = np.dtype(dtype)
        if dt == np.dtype(np.float32):
            dt = np.dtype(np.complex64)
        if dt == np.dtype(np.float64):
            dt = np.dtype(np.complex128)
        if dt not in _DTYPES:
            raise TypeError("FftPlanner accelerates f32 and f64 only (src/avx/avx_planner.rs:149-163)")
        self._precision = _DTYPES[dt]
        self._lib = lib if lib is not None else default_library()
        if self._lib.device_count() <= 0:
            raise FftError(-2, "no sm_90 CUDA device is visible (there is no CPU fallback)")
        self.device = device
        self._cache: Dict[Tuple[int, int], Fft] = {}
        self._lock = threading.Lock()

    def plan_fft(self, len: int, direction: FftDirection) -> Fft:
        key = (int(len), int(direction))
        with self._lock:
            fft = self._cache.get(key)
            if fft is None:
                fft = Fft(self._lib, int(len), FftDirection(direction), self._precision, self.device)
                self._cache[key] = fft
            return fft

    def plan_fft_with_recipe(self, recipe: Recipe, direction: FftDirection) -> Fft:
        """Planning owned by the caller: build exactly the decomposition `recipe` names (not cached)."""
        return Fft(self._lib, recipe.len, FftDirection(direction), self._precision, self.device, recipe=recipe)

    def plan_fft_2d(self, height: int, width: int, direction: FftDirection = FftDirection.Forward) -> Fft2d:
        """2-D transform of [height][width] images: the width-point plan over the rows, one strided pass down the columns."""
        return Fft2d(self._lib, height, width, direction, self._precision, self.device)

    def plan_fft_3d(self, depth: int, height: int, width: int, direction: FftDirection = FftDirection.Forward) -> "Fft3d":
        """3-D transform of [depth][height][width] volumes: the width-point plan over the rows, then one strided pass down each of
        the other two axes (not cached, like plan_fft_2d)."""
        return Fft3d(self._lib, depth, height, width, direction, self._precision, self.device)

    def plan_convolution(self, filter, signal_len: int, mode: str = "full") -> "FftConvolution":
        """Convolution of complex rows of signal_len samples with `filter` (1-D, 1..2048 taps); see FftConvolution (not cached:
        the filter is data)."""
        return FftConvolution(self._lib, filter, signal_len, mode, False, self._precision, self.device)

    def plan_channel_convolution(self, filters, signal_len: int, mode: str = "full", shared_input: bool = False) -> "ChannelConvolution":
        """Convolution of complex rows with one of C complex filters each (`filters`: [C][m], 1..2048 taps; 1-D is C = 1): per
        channel, or a filter bank over shared input rows when shared_input; see ChannelConvolution (not cached: the filters are
        data)."""
        return ChannelConvolution(self._lib, filters, signal_len, mode, shared_input, False, self._precision, self.device)


    def plan_czt(self, n: int, m: Optional[int] = None, start: float = 0.0, step: Optional[float] = None) -> "Czt":
        """Chirp-z transform of complex rows of n samples onto m points of the unit circle (default m = n), starting at `start` turns and
        `step` turns apart (default 1/m, scipy's default w); see Czt (not cached)."""
        m = int(n if m is None else m)
        return Czt(self._lib, n, m, start, 1.0 / m if step is None else step, False, self._precision, self.device)

    def plan_zoom_fft(self, n: int, fn, m: Optional[int] = None, fs: float = 2, endpoint: bool = False) -> "Czt":
        """scipy.signal.ZoomFFT(n, fn, m, fs=fs, endpoint=endpoint) for complex rows: m points (default n) of the band fn = [f1, f2]
        (a scalar fn is [0, fn]) of a signal sampled at fs; see Czt."""
        return _zoom_fft(self, n, fn, m, fs, endpoint)

    def plan_fft_forward(self, len: int) -> Fft:
        return self.plan_fft(len, FftDirection.Forward)

    def plan_fft_inverse(self, len: int) -> Fft:
        return self.plan_fft(len, FftDirection.Inverse)


class Fft2d:
    """2-D complex transform of row-major [height][width] images (a batch of them, contiguous): unnormalised, forward sign as in 1-D.
    numpy arrays go through the synchronous host entry point (in place), torch CUDA tensors through the device one (in place or into
    `out`, asynchronous on torch's current stream)."""

    def __init__(self, lib: Library, height: int, width: int, direction: FftDirection, precision: int, device: int):
        self._lib, self.height, self.width, self._precision, self.device = lib, int(height), int(width), precision, device
        self._direction = FftDirection(direction)
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_plan2d_create(ctypes.byref(self._h), self.height, self.width, int(direction), precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_plan2d_destroy(h)
            except Exception:
                pass

    def fft_direction(self) -> FftDirection:
        return self._direction

    def process(self, buffer: np.ndarray) -> None:
        want = np.complex64 if self._precision == F32 else np.complex128
        if buffer.dtype != want or not buffer.flags.c_contiguous or not buffer.flags.writeable:
            raise TypeError(f"Fft2d.process wants a contiguous writable {np.dtype(want)} array")
        per = self.height * self.width
        if buffer.size % per:
            raise FftError(-5, f"Input FFT buffer must be a multiple of FFT length. Expected multiple of {per}, got len = {buffer.size}")
        self._lib.check(self._lib.c.b200fft_exec2d_host(self._h, buffer.ctypes.data, buffer.ctypes.data, buffer.size // per))

    def process_device(self, x, out=None):
        import torch

        want = torch.complex64 if self._precision == F32 else torch.complex128
        dst = x if out is None else out
        if x.dtype != want or dst.dtype != want or not x.is_cuda or not x.is_contiguous() or not dst.is_contiguous() or dst.numel() != x.numel():
            raise TypeError(f"Fft2d.process_device wants contiguous CUDA tensors of {want} with equal sizes")
        per = self.height * self.width
        if x.numel() % per:
            raise FftError(-5, f"Input FFT buffer must be a multiple of FFT length. Expected multiple of {per}, got len = {x.numel()}")
        self._lib.check(self._lib.c.b200fft_exec2d_device(self._h, x.data_ptr(), dst.data_ptr(), x.numel() // per,
                                                          torch.cuda.current_stream(x.device).cuda_stream))
        return dst


class Fft3d:
    """3-D complex transform of row-major [depth][height][width] volumes (a batch of them, contiguous): numpy.fft.fftn over the last
    three axes, unnormalised, forward sign as in 1-D.  The width-point plan runs over the rows, then one pass down the H axis and one
    down the D axis: a compiled strided pass for power-of-two lengths up to 4096 (f64: 2048), the 2-D plans' column pass for other
    31-smooth lengths.  numpy arrays go through the synchronous host entry point (in place), torch CUDA tensors through the device one
    (in place or into `out`, asynchronous on torch's current stream).  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, depth: int, height: int, width: int, direction: FftDirection, precision: int, device: int):
        self._lib, self._precision, self.device = lib, precision, device
        self._shape = (int(depth), int(height), int(width))
        self._direction = FftDirection(direction)
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_plan3d_create(ctypes.byref(self._h), *self._shape, int(direction), precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_plan3d_destroy(h)
            except Exception:
                pass

    def fft_direction(self) -> FftDirection:
        return self._direction

    def shape(self) -> Tuple[int, int, int]:
        return self._shape

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(1024)
        rc = self._lib.c.b200fft_plan3d_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def process(self, buffer: np.ndarray) -> None:
        want = np.complex64 if self._precision == F32 else np.complex128
        if not isinstance(buffer, np.ndarray) or buffer.dtype != want or not buffer.flags.c_contiguous or not buffer.flags.writeable:
            raise TypeError(f"Fft3d.process wants a contiguous writable {np.dtype(want)} array")
        per = self._shape[0] * self._shape[1] * self._shape[2]
        if buffer.size % per:
            raise FftError(-5, f"Input FFT buffer must be a multiple of FFT length. Expected multiple of {per}, got len = {buffer.size}")
        self._lib.check(self._lib.c.b200fft_exec3d_host(self._h, buffer.ctypes.data, buffer.ctypes.data, buffer.size // per))

    def process_device(self, x, out=None):
        import torch

        want = torch.complex64 if self._precision == F32 else torch.complex128
        dst = x if out is None else out
        if x.dtype != want or dst.dtype != want or not x.is_cuda or not x.is_contiguous() or not dst.is_contiguous() or dst.numel() != x.numel():
            raise TypeError(f"Fft3d.process_device wants contiguous CUDA tensors of {want} with equal sizes")
        per = self._shape[0] * self._shape[1] * self._shape[2]
        if x.numel() % per:
            raise FftError(-5, f"Input FFT buffer must be a multiple of FFT length. Expected multiple of {per}, got len = {x.numel()}")
        self._lib.check(self._lib.c.b200fft_exec3d_device(self._h, x.data_ptr(), dst.data_ptr(), x.numel() // per,
                                                          torch.cuda.current_stream(x.device).cuda_stream))
        return dst


def _run_real(lib: Library, handle, precision: int, name: str, prefix: str, n: int, h: int, inverse: bool, src, dst):
    """Type and size checks and dispatch of the real transforms (RealFft, RealFft2d): n reals <-> h complex values per transform,
    C entry points <prefix>_{forward,inverse}_{host,device}."""
    rdt, cdt = (np.float32, np.complex64) if precision == F32 else (np.float64, np.complex128)
    sdt, ddt, sper, dper = (cdt, rdt, h, n) if inverse else (rdt, cdt, n, h)
    kind = "inverse" if inverse else "forward"
    if isinstance(src, np.ndarray):
        if src.dtype != sdt or dst.dtype != ddt or not src.flags.c_contiguous or not dst.flags.c_contiguous or not dst.flags.writeable:
            raise TypeError(f"{name} wants contiguous {np.dtype(sdt)} input and writable {np.dtype(ddt)} output")
        if src.size % sper or dst.size != src.size // sper * dper:
            raise FftError(-6, f"{name}: input holds {src.size} elements, output {dst.size}: expected batch * {sper} and batch * {dper}")
        lib.check(getattr(lib.c, f"{prefix}_{kind}_host")(handle, src.ctypes.data, dst.ctypes.data, src.size // sper))
        return dst
    import torch

    tmap = {np.float32: torch.float32, np.float64: torch.float64, np.complex64: torch.complex64, np.complex128: torch.complex128}
    if src.dtype != tmap[sdt] or dst.dtype != tmap[ddt] or not src.is_cuda or not dst.is_cuda or not src.is_contiguous() or not dst.is_contiguous():
        raise TypeError(f"{name} wants contiguous CUDA tensors of the plan's real / complex dtypes")
    if src.numel() % sper or dst.numel() != src.numel() // sper * dper:
        raise FftError(-6, f"{name}: input holds {src.numel()} elements, output {dst.numel()}: expected batch * {sper} and batch * {dper}")
    lib.check(getattr(lib.c, f"{prefix}_{kind}_device")(handle, src.data_ptr(), dst.data_ptr(), src.numel() // sper,
                                                         torch.cuda.current_stream(src.device).cuda_stream))
    return dst


class RealFft:
    """Real-to-complex / complex-to-real transforms of one even length (the shape of the `realfft` crate's RealToComplex /
    ComplexToReal on top of RustFFT's Fft; SURVEY 8(f).4).  forward: batch * len reals -> batch * (len/2 + 1) complex;
    inverse: the reverse, unnormalised (inverse(forward(x)) == len * x), equal to len * numpy.fft.irfft(X, len) for any X: the
    imaginary parts of X[0] and X[len/2] are ignored, as numpy ignores them.  numpy arrays go through the synchronous host entry
    points, torch CUDA tensors through the device ones (asynchronous on torch's current stream)."""

    def __init__(self, lib: Library, length: int, precision: int, device: int):
        self._lib, self._len, self._precision, self.device = lib, int(length), precision, device
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_real_plan_create(ctypes.byref(self._h), self._len, precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_real_plan_destroy(h)
            except Exception:
                pass

    def len(self) -> int:
        return self._len

    def complex_len(self) -> int:
        return self._len // 2 + 1

    def _run(self, inverse: bool, src, dst):
        return _run_real(self._lib, self._h, self._precision, "RealFft", "b200fft_real", self._len, self._len // 2 + 1, inverse, src, dst)

    def forward(self, real_in, complex_out):
        return self._run(False, real_in, complex_out)

    def inverse(self, complex_in, real_out):
        return self._run(True, complex_in, real_out)


class RealFft2d:
    """2-D real-to-complex / complex-to-real transforms of row-major [height][width] real images (a batch of them, contiguous), even
    width: numpy.fft.rfft2 / irfft2 over the last two axes.  forward: batch * height * width reals -> batch * height *
    (width/2 + 1) complex, unnormalised; inverse: the reverse, unnormalised (inverse(forward(x)) == height * width * x), equal to
    height * width * numpy.fft.irfft2(X, s=(height, width)) for any half spectrum X (of columns 0 and width/2 only the Hermitian
    parts count, as in numpy).  Two passes
    over half-size complex data: the width/2-point complex plan over the rows, one column pass with the real unpack / pack fused
    into its load.  Out of place only.  numpy arrays go through the synchronous host entry points, torch CUDA tensors through the
    device ones (asynchronous on torch's current stream).  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, height: int, width: int, precision: int, device: int):
        self._lib, self._height, self._width, self._precision, self.device = lib, int(height), int(width), precision, device
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_real_plan2d_create(ctypes.byref(self._h), self._height, self._width, precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_real_plan2d_destroy(h)
            except Exception:
                pass

    def height(self) -> int:
        return self._height

    def width(self) -> int:
        return self._width

    def complex_width(self) -> int:
        return self._width // 2 + 1

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_real_plan2d_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _run(self, inverse: bool, src, dst):
        return _run_real(self._lib, self._h, self._precision, "RealFft2d", "b200fft_real2d", self._height * self._width,
                         self._height * self.complex_width(), inverse, src, dst)

    def forward(self, real_in, complex_out):
        return self._run(False, real_in, complex_out)

    def inverse(self, complex_in, real_out):
        return self._run(True, complex_in, real_out)


class RealFft3d:
    """3-D real-to-complex / complex-to-real transforms of row-major [depth][height][width] real volumes (a batch of them, contiguous),
    even width: numpy.fft.rfftn / irfftn over the last three axes.  forward: batch * D * H * W reals -> batch * D * H * (W/2 + 1)
    complex, unnormalised; inverse: the reverse, unnormalised (inverse(forward(x)) == D * H * W * x), equal to
    D * H * W * numpy.fft.irfftn(X, s=(D, H, W)) for any half spectrum X.  The 2-D real transform of every [H][W] slice, then one pass
    down the D axis (the inverse: the D axis into a workspace first, so the input is never written); depth 1 is exactly RealFft2d.
    Out of place only.  numpy arrays go through the synchronous host entry points, torch CUDA tensors through the device ones
    (asynchronous on torch's current stream).  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, depth: int, height: int, width: int, precision: int, device: int):
        self._lib, self._precision, self.device = lib, precision, device
        self._depth, self._height, self._width = int(depth), int(height), int(width)
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_real_plan3d_create(ctypes.byref(self._h), self._depth, self._height, self._width, precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_real_plan3d_destroy(h)
            except Exception:
                pass

    def depth(self) -> int:
        return self._depth

    def height(self) -> int:
        return self._height

    def width(self) -> int:
        return self._width

    def complex_width(self) -> int:
        return self._width // 2 + 1

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(1024)
        rc = self._lib.c.b200fft_real_plan3d_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _run(self, inverse: bool, src, dst):
        dh = self._depth * self._height
        return _run_real(self._lib, self._h, self._precision, "RealFft3d", "b200fft_real3d", dh * self._width, dh * self.complex_width(),
                         inverse, src, dst)

    def forward(self, real_in, complex_out):
        return self._run(False, real_in, complex_out)

    def inverse(self, complex_in, real_out):
        return self._run(True, complex_in, real_out)


class RealFftPlanner:
    """Plans RealFft instances (cached per length), like realfft::RealFftPlanner over rustfft::FftPlanner."""

    def __init__(self, dtype=np.float32, device: int = 0, lib: Optional[Library] = None):
        dt = np.dtype(dtype)
        if dt in (np.dtype(np.float32), np.dtype(np.complex64)):
            self._precision = F32
        elif dt in (np.dtype(np.float64), np.dtype(np.complex128)):
            self._precision = F64
        else:
            raise TypeError("RealFftPlanner accelerates f32 and f64 only")
        self._lib = lib if lib is not None else default_library()
        if self._lib.device_count() <= 0:
            raise FftError(-2, "no sm_90 CUDA device is visible (there is no CPU fallback)")
        self.device = device
        self._cache: Dict[int, RealFft] = {}
        self._cache_2d: Dict[Tuple[int, int], RealFft2d] = {}
        self._cache_3d: Dict[Tuple[int, int, int], RealFft3d] = {}
        self._cache_hilbert: Dict[int, Hilbert] = {}
        self._lock = threading.Lock()

    def plan_fft(self, len: int) -> RealFft:
        with self._lock:
            f = self._cache.get(int(len))
            if f is None:
                f = self._cache[int(len)] = RealFft(self._lib, int(len), self._precision, self.device)
            return f

    def plan_fft_2d(self, height: int, width: int) -> RealFft2d:
        """2-D real transform of [height][width] images (even width), cached per shape; see RealFft2d."""
        key = (int(height), int(width))
        with self._lock:
            f = self._cache_2d.get(key)
            if f is None:
                f = self._cache_2d[key] = RealFft2d(self._lib, key[0], key[1], self._precision, self.device)
            return f

    def plan_fft_3d(self, depth: int, height: int, width: int) -> RealFft3d:
        """3-D real transform of [depth][height][width] volumes (even width), cached per shape; see RealFft3d."""
        key = (int(depth), int(height), int(width))
        with self._lock:
            f = self._cache_3d.get(key)
            if f is None:
                f = self._cache_3d[key] = RealFft3d(self._lib, key[0], key[1], key[2], self._precision, self.device)
            return f

    def plan_hilbert(self, len: int) -> "Hilbert":
        """Analytic signal (scipy.signal.hilbert) of real rows of `len` samples, cached per length; see Hilbert."""
        with self._lock:
            h = self._cache_hilbert.get(int(len))
            if h is None:
                h = self._cache_hilbert[int(len)] = Hilbert(self._lib, int(len), self._precision, self.device)
            return h

    def plan_convolution(self, filter, signal_len: int, mode: str = "full") -> FftConvolution:
        """Convolution of real rows of signal_len samples with the real `filter` (1-D, 1..2048 taps); see FftConvolution (not
        cached: the filter is data)."""
        return FftConvolution(self._lib, filter, signal_len, mode, True, self._precision, self.device)

    def plan_channel_convolution(self, filters, signal_len: int, mode: str = "full", shared_input: bool = False) -> "ChannelConvolution":
        """Convolution of real rows with one of C real filters each (`filters`: [C][m], 1..2048 taps; 1-D is C = 1): per channel, or
        a filter bank over shared input rows when shared_input; see ChannelConvolution (not cached: the filters are data)."""
        return ChannelConvolution(self._lib, filters, signal_len, mode, shared_input, True, self._precision, self.device)

    def plan_convolution_2d(self, filter, image_shape, mode: str = "full") -> "FftConvolution2d":
        """2-D convolution of real images of image_shape = (height, width) with the real 2-D `filter`; see FftConvolution2d (not
        cached: the filter is data)."""
        return FftConvolution2d(self._lib, filter, image_shape, mode, self._precision, self.device)

    def plan_stft(self, window, hop: int, signal_len: int, center: bool = True) -> "Stft":
        """Short-time Fourier transform of real rows of signal_len samples with the real 1-D `window` (its length is n_fft) and
        `hop`; see Stft (not cached: the window is data)."""
        return Stft(self._lib, window, hop, signal_len, center, self._precision, self.device)

    def plan_czt(self, n: int, m: Optional[int] = None, start: float = 0.0, step: Optional[float] = None) -> "Czt":
        """Chirp-z transform of real rows of n samples onto m points of the unit circle (default m = n), starting at `start` turns and
        `step` turns apart (default 1/m, scipy's default w); see Czt (not cached)."""
        m = int(n if m is None else m)
        return Czt(self._lib, n, m, start, 1.0 / m if step is None else step, True, self._precision, self.device)

    def plan_zoom_fft(self, n: int, fn, m: Optional[int] = None, fs: float = 2, endpoint: bool = False) -> "Czt":
        """scipy.signal.ZoomFFT(n, fn, m, fs=fs, endpoint=endpoint) for real rows: m points (default n) of the band fn = [f1, f2]
        (a scalar fn is [0, fn]) of a signal sampled at fs; see Czt."""
        return _zoom_fft(self, n, fn, m, fs, endpoint)


class Stft:
    """Batched short-time Fourier transform of real rows with one window, hop, signal length and `center` fixed at plan time.
    forward: batch * signal_len reals -> batch * frames * (n_fft/2 + 1) complex values, frame-major (row r, frame f, bin k at
    (r frames + f) bins + k), unnormalised:

        S[f][k] = sum_u w[u] xp[f hop + u] exp(-2 pi i k u / n_fft)

    with xp the row reflect-padded by n_fft/2 on each side when center, so that S equals torch.stft(x, n_fft, hop, window=w,
    center=center, pad_mode="reflect", return_complex=True).transpose(-2, -1).  inverse: the least-squares inverse, equal to
    torch.istft(S.transpose(-2, -1), n_fft, hop, window=w, center=center, length=signal_len), so inverse(forward(x)) = x.  Unlike the
    library's other transforms the inverse is normalised: the division by the window envelope sum_f w[t - f hop]^2 is part of an
    inverse STFT, and the 1/n_fft folds into the same multiply.  It ignores the imaginary parts of bins 0 and n_fft/2, as numpy's
    irfft does, and needs the NOLA condition (envelope > 1e-11 at every returned sample): a plan that fails it still runs forward,
    and its inverse raises FftError (B200FFT_ERR_UNSUPPORTED).  Power-of-two n_fft from 4 to 32768 (f64: 16384) run the forward in
    one pass; other even n_fft frame into a workspace and run the real plan.  Out of place only.  numpy arrays go through the
    synchronous host entry points, torch CUDA tensors through the device ones (asynchronous on torch's current stream).  Immutable
    and safe to call from many threads."""

    def __init__(self, lib: Library, window, hop: int, signal_len: int, center: bool, precision: int, device: int):
        self._lib, self._precision, self.device = lib, precision, device
        self._hop, self._signal_len, self._center = int(hop), int(signal_len), bool(center)
        if np.iscomplexobj(window):
            raise TypeError("an STFT plan needs a real window")
        w = np.ascontiguousarray(np.asarray(window), dtype=self.real_dtype)
        if w.ndim != 1:
            raise TypeError("the window must be 1-D")
        self._n_fft = int(w.size)
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_stft_plan_create(ctypes.byref(self._h), self._signal_len, w.ctypes.data, self._n_fft, self._hop,
                                                 1 if self._center else 0, precision, device))
        self._frames = int(lib.c.b200fft_stft_frames(self._h))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_stft_plan_destroy(h)
            except Exception:
                pass

    @property
    def real_dtype(self):
        return np.float32 if self._precision == F32 else np.float64

    @property
    def complex_dtype(self):
        return np.complex64 if self._precision == F32 else np.complex128

    def n_fft(self) -> int:
        return self._n_fft

    def hop(self) -> int:
        return self._hop

    def signal_len(self) -> int:
        return self._signal_len

    def center(self) -> bool:
        return self._center

    def frames(self) -> int:
        return self._frames

    def bins(self) -> int:
        return self._n_fft // 2 + 1

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_stft_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _run(self, inverse: bool, src, dst):
        return _run_real(self._lib, self._h, self._precision, "Stft", "b200fft_stft", self._signal_len, self._frames * self.bins(), inverse,
                         src, dst)

    def forward(self, x, spec):
        """Every row of `x` (batch * signal_len reals) into `spec` (batch * frames * bins complex values, any shape); returns `spec`."""
        return self._run(False, x, spec)

    def inverse(self, spec, y):
        """Every row of spectra in `spec` (batch * frames * bins complex values) into `y` (batch * signal_len reals); returns `y`."""
        return self._run(True, spec, y)


def _zoom_fft(planner, n: int, fn, m: Optional[int], fs: float, endpoint: bool) -> "Czt":
    f = np.atleast_1d(np.asarray(fn, dtype=np.float64))
    if f.shape == (1,):
        f1, f2 = 0.0, float(f[0])
    elif f.shape == (2,):
        f1, f2 = float(f[0]), float(f[1])
    else:
        raise ValueError("fn must be a scalar or a sequence of two frequencies [f1, f2]")
    m = int(n if m is None else m)
    if endpoint and m < 2:
        raise ValueError("a zoom FFT with endpoint=True needs m >= 2 points")
    return planner.plan_czt(n, m, f1 / fs, (f2 - f1) / (fs * (m - 1 if endpoint else m)))


class Czt:
    """Batched chirp-z transform on the unit circle with n, m, start and step fixed at plan time.  Every contiguous row x of n samples
    becomes m complex values, unnormalised:

        y[k] = sum_{t<n} x[t] exp(-2 pi i (start + k step) t),   k = 0 .. m - 1

    with start and step in turns (cycles per sample).  This is scipy.signal.czt(x, m, w=exp(-2j pi step), a=exp(2j pi start)); a
    caller holding scipy's unit-modulus w and a converts with step = -angle(w) / (2 pi) and start = angle(a) / (2 pi).  A zoom FFT
    of the band [f1, f2] of a signal sampled at fs is start = f1 / fs, step = (f2 - f1) / (fs m) (endpoint: / (fs (m - 1))):
    FftPlanner.plan_zoom_fft.  Spirals (|w| != 1 or |a| != 1) are not supported.  The tables use the exact phase of start and
    step (reduced mod 1 in integers, not formed in double as scipy does), so the error stays at FFT level up to n + m - 1 = 2^24.

    Complex rows from FftPlanner.plan_czt, real rows from RealFftPlanner.plan_czt (the output is complex either way).
    max(8, next_pow2(n + m - 1)) <= 4096 runs in one pass (one read of x, one write of y); longer transforms run a pre-chirp pass,
    the library's power-of-two forward and inverse plans and a post-chirp pass on a workspace.  Out of place only.  numpy arrays
    go through the synchronous host entry point, torch CUDA tensors through the device one (asynchronous on torch's current
    stream).  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, n: int, m: int, start: float, step: float, real: bool, precision: int, device: int):
        self._lib, self._real, self._precision, self.device = lib, bool(real), precision, device
        self._n, self._m, self._start, self._step = int(n), int(m), float(start), float(step)
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_czt_plan_create(ctypes.byref(self._h), self._n, self._m, self._start, self._step, 1 if real else 0,
                                                precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_czt_plan_destroy(h)
            except Exception:
                pass

    @property
    def dtype(self):
        """dtype of the input rows."""
        if self._real:
            return np.float32 if self._precision == F32 else np.float64
        return self.out_dtype

    @property
    def out_dtype(self):
        return np.complex64 if self._precision == F32 else np.complex128

    def n(self) -> int:
        return self._n

    def m(self) -> int:
        return self._m

    def start(self) -> float:
        return self._start

    def step(self) -> float:
        return self._step

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_czt_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n_in: int, n_out: int) -> int:
        if n_in % self._n or n_out != n_in // self._n * self._m:
            raise FftError(-6, f"Czt: input holds {n_in} samples, output {n_out}: expected batch * {self._n} and batch * {self._m}")
        return n_in // self._n

    def process(self, x, out):
        """Transform every row of `x` (batch * n samples) into `out` (batch * m complex values, any shape); returns `out`."""
        if isinstance(x, np.ndarray):
            want, wout = np.dtype(self.dtype), np.dtype(self.out_dtype)
            if not isinstance(out, np.ndarray) or x.dtype != want or out.dtype != wout or not x.flags.c_contiguous \
                    or not out.flags.c_contiguous or not out.flags.writeable:
                raise TypeError(f"Czt wants contiguous {want.name} input and a writable contiguous {wout.name} output")
            batch = self._batch(x.size, out.size)
            self._lib.check(self._lib.c.b200fft_czt_host(self._h, x.ctypes.data, out.ctypes.data, batch))
            return out
        import torch

        tmap = {np.float32: torch.float32, np.float64: torch.float64, np.complex64: torch.complex64, np.complex128: torch.complex128}
        want, wout = tmap[self.dtype], tmap[self.out_dtype]
        if not isinstance(out, torch.Tensor) or x.dtype != want or out.dtype != wout or not x.is_cuda or not out.is_cuda \
                or not x.is_contiguous() or not out.is_contiguous():
            raise TypeError(f"Czt wants contiguous CUDA tensors of {want} (input) and {wout} (output)")
        if x.device.index != self.device or out.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{out.device.index}, plan is on cuda:{self.device}")
        batch = self._batch(x.numel(), out.numel())
        self._lib.check(self._lib.c.b200fft_czt_device(self._h, x.data_ptr(), out.data_ptr(), batch,
                                                       torch.cuda.current_stream(x.device).cuda_stream))
        return out


class Hilbert:
    """Batched analytic signal of real rows, scipy.signal.hilbert(x, axis=-1): every contiguous row x of len() reals becomes len()
    complex values z = x + i y, with y the Hilbert transform of x,

        z = ifft(fft(x) h),   h = 1, 2, ..., 2, (1 at N/2 for even N), 0, ...

    Normalised, unlike the library's FFTs: the real part of z is x itself, bit for bit.  |z| is the envelope and angle(z) the
    instantaneous phase.  Power-of-two lengths from 4 to 32768 (f64: 16384) run in one pass (one read of x, one write of z); other
    even lengths run the len/2-point complex plans on a workspace, odd lengths the len-point plans in the output itself.  Even
    lengths read x as pairs, so a CUDA tensor input must start at an even element (TypeError otherwise).  Out of place only.  numpy
    arrays go through the synchronous host entry point, torch CUDA tensors through the device one (asynchronous on torch's
    current stream).  From RealFftPlanner.plan_hilbert.  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, length: int, precision: int, device: int):
        self._lib, self._len, self._precision, self.device = lib, int(length), precision, device
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_hilbert_plan_create(ctypes.byref(self._h), self._len, precision, device))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_hilbert_plan_destroy(h)
            except Exception:
                pass

    def len(self) -> int:
        return self._len

    @property
    def dtype(self):
        """dtype of the input rows."""
        return np.float32 if self._precision == F32 else np.float64

    @property
    def out_dtype(self):
        return np.complex64 if self._precision == F32 else np.complex128

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_hilbert_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n_in: int, n_out: int) -> int:
        if n_in != n_out or (self._len and n_in % self._len) or (not self._len and n_in):
            raise FftError(-6, f"Hilbert: input holds {n_in} samples, output {n_out}: expected batch * {self._len} each")
        return n_in // self._len if self._len else 0

    def process(self, x, out):
        """Every row of `x` (batch * len() reals) into `out` (batch * len() complex values, any shape); returns `out`."""
        if isinstance(x, np.ndarray):
            want, wout = np.dtype(self.dtype), np.dtype(self.out_dtype)
            if not isinstance(out, np.ndarray) or x.dtype != want or out.dtype != wout or not x.flags.c_contiguous \
                    or not out.flags.c_contiguous or not out.flags.writeable:
                raise TypeError(f"Hilbert wants contiguous {want.name} input and a writable contiguous {wout.name} output")
            batch = self._batch(x.size, out.size)
            self._lib.check(self._lib.c.b200fft_hilbert_host(self._h, x.ctypes.data, out.ctypes.data, batch))
            return out
        import torch

        want = torch.float32 if self._precision == F32 else torch.float64
        wout = torch.complex64 if self._precision == F32 else torch.complex128
        if not isinstance(out, torch.Tensor) or x.dtype != want or out.dtype != wout or not x.is_cuda or not out.is_cuda \
                or not x.is_contiguous() or not out.is_contiguous():
            raise TypeError(f"Hilbert wants contiguous CUDA tensors of {want} (input) and {wout} (output)")
        if x.device.index != self.device or out.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{out.device.index}, plan is on cuda:{self.device}")
        if self._len % 2 == 0 and x.data_ptr() % (2 * x.element_size()):
            raise TypeError("Hilbert.process: even lengths read x as pairs, so the input tensor must start at an even element")
        batch = self._batch(x.numel(), out.numel())
        self._lib.check(self._lib.c.b200fft_hilbert_device(self._h, x.data_ptr(), out.data_ptr(), batch,
                                                           torch.cuda.current_stream(x.device).cuda_stream))
        return out


class FftConvolution:
    """Batched FFT convolution with one filter fixed at plan time: every contiguous row of signal_len samples becomes
    scipy.signal.fftconvolve(row, filter, mode) -- plain sums, no scaling.  mode "full" (signal_len + m - 1 outputs), "same"
    (signal_len, scipy's centring) or "valid" (signal_len - m + 1, needs signal_len >= m).  Complex rows and filter from
    FftPlanner.plan_convolution, real ones from RealFftPlanner.plan_convolution.  Cross-correlation with h is the convolution
    with np.conj(h[::-1]).

    One launch and one pass over device memory (overlap-save inside one CTA per block), out of place only.  numpy arrays go
    through the synchronous host entry point, torch CUDA tensors through the device one (asynchronous on torch's current
    stream).  Immutable and safe to call from many threads."""

    MODES = {"full": 0, "same": 1, "valid": 2}

    def __init__(self, lib: Library, filter, signal_len: int, mode: str, real: bool, precision: int, device: int):
        if mode not in self.MODES:
            raise FftError(-1, f"unknown convolution mode {mode!r}: expected one of {sorted(self.MODES)}")
        self._lib, self._real, self._precision, self.device, self.mode = lib, bool(real), precision, device, mode
        self._signal_len = int(signal_len)
        if real and np.iscomplexobj(filter):
            raise TypeError("a real convolution plan needs a real filter")
        h = np.ascontiguousarray(np.asarray(filter), dtype=self.dtype)
        if h.ndim != 1:
            raise TypeError("the filter must be 1-D")
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_conv_plan_create(ctypes.byref(self._h), self._signal_len, h.ctypes.data, h.size, self.MODES[mode],
                                                 1 if real else 0, precision, device))
        self._out_len = int(lib.c.b200fft_conv_output_len(self._h))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_conv_plan_destroy(h)
            except Exception:
                pass

    @property
    def dtype(self):
        if self._real:
            return np.float32 if self._precision == F32 else np.float64
        return np.complex64 if self._precision == F32 else np.complex128

    def signal_len(self) -> int:
        return self._signal_len

    def output_len(self) -> int:
        return self._out_len

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(256)
        rc = self._lib.c.b200fft_conv_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n_in: int, n_out: int) -> int:
        n, o = self._signal_len, self._out_len
        if n == 0:
            return 0
        if n_in % n or n_out != n_in // n * o:
            raise FftError(-6, f"FftConvolution: input holds {n_in} samples, output {n_out}: expected batch * {n} and batch * {o}")
        return n_in // n

    def process(self, x, out):
        """Convolve every row of `x` (batch * signal_len samples) into `out` (batch * output_len samples); returns `out`."""
        if isinstance(x, np.ndarray):
            want = np.dtype(self.dtype)
            if not isinstance(out, np.ndarray) or x.dtype != want or out.dtype != want or not x.flags.c_contiguous \
                    or not out.flags.c_contiguous or not out.flags.writeable:
                raise TypeError(f"FftConvolution wants contiguous {want.name} input and a writable {want.name} output")
            batch = self._batch(x.size, out.size)
            self._lib.check(self._lib.c.b200fft_conv_host(self._h, x.ctypes.data, out.ctypes.data, batch))
            return out
        import torch

        tmap = {np.float32: torch.float32, np.float64: torch.float64, np.complex64: torch.complex64, np.complex128: torch.complex128}
        want = tmap[self.dtype]
        if not isinstance(out, torch.Tensor) or x.dtype != want or out.dtype != want or not x.is_cuda or not out.is_cuda \
                or not x.is_contiguous() or not out.is_contiguous():
            raise TypeError(f"FftConvolution wants contiguous CUDA tensors of {want}")
        if x.device.index != self.device or out.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{out.device.index}, plan is on cuda:{self.device}")
        batch = self._batch(x.numel(), out.numel())
        self._lib.check(self._lib.c.b200fft_conv_device(self._h, x.data_ptr(), out.data_ptr(), batch,
                                                        torch.cuda.current_stream(x.device).cuda_stream))
        return out


class ChannelConvolution:
    """Batched multi-channel FFT convolution with C filters of m taps fixed at plan time.  The output is batch * C rows of
    output_len samples, row (b, c) at (b C + c) output_len, and every row is scipy.signal.fftconvolve(input row, filters[c], mode)
    -- plain sums, no scaling, modes and output lengths as for FftConvolution:
      per channel (default)  input [batch][C][signal_len]:  y[b][c] = x[b][c] (*) h[c]
                             = scipy.signal.fftconvolve(x, h[None], mode, axes=-1)
      shared_input=True      input [batch][signal_len], a filter bank over each row:  y[b][c] = x[b] (*) h[c]
                             = scipy.signal.fftconvolve(np.broadcast_to(x[:, None, :], (batch, C, signal_len)), h[None], mode,
                             axes=-1)  (without the broadcast, scipy's "same" crops the channel axis to 1)
    Complex rows and filters from FftPlanner.plan_channel_convolution, real ones from RealFftPlanner.plan_channel_convolution.
    C = 1 (a 1-D filters array) computes exactly what FftConvolution does.

    One launch and one pass over device memory (overlap-save inside one CTA per block), out of place only.  numpy arrays go
    through the synchronous host entry point, torch CUDA tensors through the device one (asynchronous on torch's current
    stream).  Immutable and safe to call from many threads."""

    MODES = FftConvolution.MODES

    def __init__(self, lib: Library, filters, signal_len: int, mode: str, shared: bool, real: bool, precision: int, device: int):
        if mode not in self.MODES:
            raise FftError(-1, f"unknown convolution mode {mode!r}: expected one of {sorted(self.MODES)}")
        self._lib, self._real, self._precision, self.device, self.mode = lib, bool(real), precision, device, mode
        self._shared, self._signal_len = bool(shared), int(signal_len)
        if real and np.iscomplexobj(filters):
            raise TypeError("a real convolution plan needs real filters")
        h = np.ascontiguousarray(np.asarray(filters), dtype=self.dtype)
        if h.ndim == 1:
            h = h[None]
        if h.ndim != 2:
            raise TypeError("the filters must be 1-D or 2-D ([channels][taps])")
        self._channels = int(h.shape[0])
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_chconv_plan_create(ctypes.byref(self._h), self._signal_len, self._channels, h.ctypes.data, h.shape[1],
                                                   self.MODES[mode], 1 if real else 0, 1 if shared else 0, precision, device))
        self._out_len = int(lib.c.b200fft_chconv_output_len(self._h))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_chconv_plan_destroy(h)
            except Exception:
                pass

    @property
    def dtype(self):
        if self._real:
            return np.float32 if self._precision == F32 else np.float64
        return np.complex64 if self._precision == F32 else np.complex128

    def channels(self) -> int:
        return self._channels

    def signal_len(self) -> int:
        return self._signal_len

    def output_len(self) -> int:
        return self._out_len

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(256)
        rc = self._lib.c.b200fft_chconv_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n_in: int, n_out: int) -> int:
        C, o = self._channels, self._out_len
        n = self._signal_len * (1 if self._shared else C)  # input samples per batch element
        if n == 0:
            return 0
        if n_in % n or n_out != n_in // n * C * o:
            raise FftError(-6, f"ChannelConvolution: input holds {n_in} samples, output {n_out}: expected batch * {n} and "
                               f"batch * {C * o}")
        return n_in // n

    def process(self, x, out):
        """Convolve every input row of `x` (batch * C * signal_len samples, or batch * signal_len with shared input) into `out`
        (batch * C * output_len samples); returns `out`."""
        if isinstance(x, np.ndarray):
            want = np.dtype(self.dtype)
            if not isinstance(out, np.ndarray) or x.dtype != want or out.dtype != want or not x.flags.c_contiguous \
                    or not out.flags.c_contiguous or not out.flags.writeable:
                raise TypeError(f"ChannelConvolution wants contiguous {want.name} input and a writable {want.name} output")
            batch = self._batch(x.size, out.size)
            self._lib.check(self._lib.c.b200fft_chconv_host(self._h, x.ctypes.data, out.ctypes.data, batch))
            return out
        import torch

        tmap = {np.float32: torch.float32, np.float64: torch.float64, np.complex64: torch.complex64, np.complex128: torch.complex128}
        want = tmap[self.dtype]
        if not isinstance(out, torch.Tensor) or x.dtype != want or out.dtype != want or not x.is_cuda or not out.is_cuda \
                or not x.is_contiguous() or not out.is_contiguous():
            raise TypeError(f"ChannelConvolution wants contiguous CUDA tensors of {want}")
        if x.device.index != self.device or out.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{out.device.index}, plan is on cuda:{self.device}")
        batch = self._batch(x.numel(), out.numel())
        self._lib.check(self._lib.c.b200fft_chconv_device(self._h, x.data_ptr(), out.data_ptr(), batch,
                                                          torch.cuda.current_stream(x.device).cuda_stream))
        return out


class FftConvolution2d:
    """Batched 2-D FFT convolution of real images with one real filter fixed at plan time: every contiguous [height][width] image
    becomes scipy.signal.fftconvolve(image, filter, mode) -- plain sums, no scaling.  mode "full" ((height + kh - 1) x
    (width + kw - 1) outputs), "same" (height x width, scipy's centring) or "valid" ((height - kh + 1) x (width - kw + 1), needs an
    image at least as large as the filter; the inputs are not swapped).  Cross-correlation with h is the convolution with
    h[::-1, ::-1].

    Three passes over half-size complex data (row FFTs, one fused column pass with the filter's spectrum, inverse row FFTs that
    store only the requested pixels), out of place only.  The padded size of the circular convolution must stay within 4096 rows
    and 4096 complex columns (f64: 2048).  numpy arrays go through the synchronous host entry point, torch CUDA tensors through the
    device one (asynchronous on torch's current stream).  Immutable and safe to call from many threads."""

    MODES = FftConvolution.MODES

    def __init__(self, lib: Library, filter, image_shape, mode: str, precision: int, device: int):
        if mode not in self.MODES:
            raise FftError(-1, f"unknown convolution mode {mode!r}: expected one of {sorted(self.MODES)}")
        self._lib, self._precision, self.device, self.mode = lib, precision, device, mode
        self._shape = tuple(int(v) for v in image_shape)
        if len(self._shape) != 2:
            raise TypeError("image_shape must be (height, width)")
        if np.iscomplexobj(filter):
            raise TypeError("a real convolution plan needs a real filter")
        h = np.ascontiguousarray(np.asarray(filter), dtype=self.dtype)
        if h.ndim != 2:
            raise TypeError("the filter must be 2-D")
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_conv2d_plan_create(ctypes.byref(self._h), self._shape[0], self._shape[1], h.ctypes.data, h.shape[0],
                                                   h.shape[1], self.MODES[mode], precision, device))
        ho, wo = ctypes.c_uint64(), ctypes.c_uint64()
        lib.check(lib.c.b200fft_conv2d_output_shape(self._h, ctypes.byref(ho), ctypes.byref(wo)))
        self._out_shape = (int(ho.value), int(wo.value))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_conv2d_plan_destroy(h)
            except Exception:
                pass

    @property
    def dtype(self):
        return np.float32 if self._precision == F32 else np.float64

    def image_shape(self) -> Tuple[int, int]:
        return self._shape

    def output_shape(self) -> Tuple[int, int]:
        return self._out_shape

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(256)
        rc = self._lib.c.b200fft_conv2d_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n_in: int, n_out: int) -> int:
        n, o = self._shape[0] * self._shape[1], self._out_shape[0] * self._out_shape[1]
        if n_in % n or n_out != n_in // n * o:
            raise FftError(-6, f"FftConvolution2d: input holds {n_in} samples, output {n_out}: expected batch * {n} and batch * {o}")
        return n_in // n

    def process(self, x, out):
        """Convolve every image of `x` (batch * height * width samples, any shape) into `out` (batch * output height * output width
        samples); returns `out`."""
        if isinstance(x, np.ndarray):
            want = np.dtype(self.dtype)
            if not isinstance(out, np.ndarray) or x.dtype != want or out.dtype != want or not x.flags.c_contiguous \
                    or not out.flags.c_contiguous or not out.flags.writeable:
                raise TypeError(f"FftConvolution2d wants contiguous {want.name} input and a writable {want.name} output")
            batch = self._batch(x.size, out.size)
            self._lib.check(self._lib.c.b200fft_conv2d_host(self._h, x.ctypes.data, out.ctypes.data, batch))
            return out
        import torch

        want = torch.float32 if self._precision == F32 else torch.float64
        if not isinstance(out, torch.Tensor) or x.dtype != want or out.dtype != want or not x.is_cuda or not out.is_cuda \
                or not x.is_contiguous() or not out.is_contiguous():
            raise TypeError(f"FftConvolution2d wants contiguous CUDA tensors of {want}")
        if x.device.index != self.device or out.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{out.device.index}, plan is on cuda:{self.device}")
        batch = self._batch(x.numel(), out.numel())
        self._lib.check(self._lib.c.b200fft_conv2d_device(self._h, x.data_ptr(), out.data_ptr(), batch,
                                                          torch.cuda.current_stream(x.device).cuda_stream))
        return out


class DctKind(enum.IntEnum):
    """The rustdct traits a plan implements (B200FFT_DCT2 ... B200FFT_DST4)."""
    Dct2 = 0
    Dct3 = 1
    Dct4 = 2
    Dst2 = 3
    Dst3 = 4
    Dst4 = 5


class Dct:
    """One planned DCT or DST of one length (the shape of rustdct's Dct2 / Dct3 / Dct4 / Dst2 / Dst3 / Dst4 over RustFFT's Fft):
    every contiguous row of len() reals is transformed, unnormalised, as scipy.fft.dct / dst(x, type) / 2:

        Dct2  X[k] = sum x[n] cos(pi (2n+1) k / 2N)             Dst2  X[k] = sum x[n] sin(pi (2n+1)(k+1) / 2N)
        Dct3  X[k] = x[0]/2 + sum_{n>=1} x[n] cos(pi n (2k+1) / 2N)
        Dst3  X[k] = (-1)^k x[N-1]/2 + sum_{n<=N-2} x[n] sin(pi (n+1)(2k+1) / 2N)
        Dct4  X[k] = sum x[n] cos(pi (2n+1)(2k+1) / 4N)         Dst4  X[k] = sum x[n] sin(pi (2n+1)(2k+1) / 4N)

    so Dct3(Dct2(x)) = Dst3(Dst2(x)) = Dct4(Dct4(x)) = Dst4(Dst4(x)) = (N/2) x.  Powers of two from 4 to 32768 (f64: 16384) run in
    one pass, which moves element pairs: its device buffers must start at an even element (a torch view such as x[1:] of an
    allocation does not; process_device raises TypeError for it).  Other lengths run around a complex plan and take any offset.  process(buffer) transforms a numpy array in place through the synchronous
    host entry point; process_device(x, out=None) takes torch CUDA tensors, in place when out is None, asynchronous on torch's
    current stream.  Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, length: int, kind: DctKind, precision: int, device: int):
        self._lib, self._len, self._kind, self._precision, self.device = lib, int(length), DctKind(kind), precision, device
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_dct_plan_create(ctypes.byref(self._h), self._len, int(kind), precision, device))
        self._fused = ",fused," in self.describe()

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_dct_plan_destroy(h)
            except Exception:
                pass

    def len(self) -> int:
        return self._len

    def __len__(self) -> int:
        return self._len

    def kind(self) -> DctKind:
        return self._kind

    @property
    def dtype(self):
        return np.float32 if self._precision == F32 else np.float64

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(512)
        rc = self._lib.c.b200fft_dct_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n: int) -> int:
        if self._len == 0:
            return 0
        if n % self._len:
            raise FftError(-5, f"Dct: buffer holds {n} samples, expected a multiple of {self._len}")
        return n // self._len

    def process(self, buffer: np.ndarray) -> np.ndarray:
        """Transform every row of `buffer` (batch * len() reals, contiguous, writable) in place; returns it."""
        want = np.dtype(self.dtype)
        if not isinstance(buffer, np.ndarray) or buffer.dtype != want or not buffer.flags.c_contiguous or not buffer.flags.writeable:
            raise TypeError(f"Dct.process wants a contiguous writable {want.name} array")
        batch = self._batch(buffer.size)
        self._lib.check(self._lib.c.b200fft_dct_host(self._h, buffer.ctypes.data, buffer.ctypes.data, batch))
        return buffer

    def process_device(self, x, out=None):
        """x: torch CUDA tensor of batch * len() reals (any shape, contiguous); in place when `out` is None.  Returns the result."""
        import torch

        want = torch.float32 if self._precision == F32 else torch.float64
        dst = x if out is None else out
        if not isinstance(dst, torch.Tensor) or x.dtype != want or dst.dtype != want or not x.is_cuda or not dst.is_cuda \
                or not x.is_contiguous() or not dst.is_contiguous():
            raise TypeError(f"Dct.process_device wants contiguous CUDA tensors of {want}")
        if x.device.index != self.device or dst.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{dst.device.index}, plan is on cuda:{self.device}")
        if dst.numel() != x.numel():
            raise FftError(-6, f"Dct: input holds {x.numel()} samples, output {dst.numel()}: expected equal sizes")
        if self._fused and (x.data_ptr() | dst.data_ptr()) % (2 * x.element_size()):
            raise TypeError("Dct.process_device: a one-pass plan needs tensors that start at an even element (it moves element pairs)")
        batch = self._batch(x.numel())
        self._lib.check(self._lib.c.b200fft_dct_device(self._h, x.data_ptr(), dst.data_ptr(), batch,
                                                       torch.cuda.current_stream(x.device).cuda_stream))
        return dst


_PI_LD = np.longdouble("3.14159265358979323846264338327950288")


def mdct_window(name: str, length: int, dtype=np.float64) -> np.ndarray:
    """rustdct's window_fn::sine / vorbis of 2 * length taps, evaluated in np.longdouble and rounded once to `dtype`:
    sine[n] = sin(pi (n + 1/2) / 2N), vorbis[n] = sin(pi/2 sin^2(pi (n + 1/2) / 2N))."""
    n = np.arange(2 * int(length), dtype=np.longdouble)
    s = np.sin(_PI_LD * (n + np.longdouble(0.5)) / np.longdouble(2 * int(length)))
    if name == "sine":
        return s.astype(dtype)
    if name == "vorbis":
        return np.sin(_PI_LD / 2 * s * s).astype(dtype)
    raise ValueError(f"unknown MDCT window {name!r}: expected 'sine', 'vorbis' or an array of 2 * len taps")


class Mdct:
    """Batched modified DCT of real rows (rustdct's Mdct) with N = len(), a real window w of 2N taps and the signal length L fixed at
    plan time.  A row x is padded with N zeros on each side and cut into frames() = ceil(L / N) + 1 frames of 2N samples at a hop of
    N; frame f covers xp[f N, f N + 2N), xp = N zeros, x, zeros.  forward: batch * L reals -> batch * frames * N reals, frame-major,
    unnormalised as rustdct defines it:

        C[f][k] = sum_{n < 2N} w[n] xp[f N + n] cos(pi/N (n + 1/2 + N/2)(k + 1/2))

    so row f equals rustdct's process_mdct(xp[fN .. fN + N], xp[fN + N .. fN + 2N]).  inverse: the overlap-add of (2/N) times
    rustdct's process_imdct of every frame, cropped to [N, N + L).  For a Princen-Bradley window (w[n]^2 + w[n + N]^2 = 1,
    w[2N - 1 - n] = w[n]: "sine", "vorbis", KBD) inverse(forward(x)) = x, the first and last N samples included; any other window
    computes the same formula.  N must be even.  Power-of-two N from 64 to 512 (f64: 64 to 16384) run the forward in one pass (the
    lengths where that pass beat the general route on an H100); other N fold into the output and run the N-point Dct4 plan on it.  The inverse runs the Dct4 plan into a workspace, then one overlap-add pass.
    When the Dct4 of N is a one-pass plan the coefficient tensor must start at an even element (TypeError otherwise).  Out of place
    only.  numpy arrays go through the synchronous host entry points (forward / inverse), torch CUDA tensors through the device ones
    (forward_device / inverse_device, asynchronous on torch's current stream).  From DctPlanner.plan_mdct.  Immutable and safe to
    call from many threads."""

    def __init__(self, lib: Library, length: int, window: np.ndarray, signal_len: int, precision: int, device: int):
        self._lib, self._len, self._signal_len, self._precision, self.device = lib, int(length), int(signal_len), precision, device
        self._h = ctypes.c_void_p()
        lib.check(lib.c.b200fft_mdct_plan_create(ctypes.byref(self._h), self._len, window.ctypes.data, self._signal_len, precision, device))
        self._frames = int(lib.c.b200fft_mdct_frames(self._h))
        self._pairs = re.search(r"(^Mdct\{[^{]*|dct=Dct4\{n=\d+),fused,", self.describe()) is not None

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_mdct_plan_destroy(h)
            except Exception:
                pass

    def len(self) -> int:
        return self._len

    def signal_len(self) -> int:
        return self._signal_len

    def frames(self) -> int:
        return self._frames

    @property
    def dtype(self):
        return np.float32 if self._precision == F32 else np.float64

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(1024)
        rc = self._lib.c.b200fft_mdct_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _host(self, kind: str, src, dst, sper: int, dper: int):
        want = np.dtype(self.dtype)
        if not isinstance(src, np.ndarray) or src.dtype != want or not src.flags.c_contiguous:
            raise TypeError(f"Mdct.{kind} wants a contiguous {want.name} array")
        if src.size % sper:
            raise FftError(-6, f"Mdct: input holds {src.size} elements, expected batch * {sper}")
        batch = src.size // sper
        if dst is None:
            dst = np.empty((batch, self._frames, self._len) if kind == "forward" else (batch, self._signal_len), want)
        if not isinstance(dst, np.ndarray) or dst.dtype != want or not dst.flags.c_contiguous or not dst.flags.writeable:
            raise TypeError(f"Mdct.{kind} wants a writable contiguous {want.name} output")
        if dst.size != batch * dper:
            raise FftError(-6, f"Mdct: output holds {dst.size} elements, expected {batch} * {dper}")
        self._lib.check(getattr(self._lib.c, f"b200fft_mdct_{kind}_host")(self._h, src.ctypes.data, dst.ctypes.data, batch))
        return dst

    def _device(self, kind: str, src, dst, sper: int, dper: int):
        import torch

        want = torch.float32 if self._precision == F32 else torch.float64
        if not isinstance(src, torch.Tensor) or src.dtype != want or not src.is_cuda or not src.is_contiguous():
            raise TypeError(f"Mdct.{kind}_device wants a contiguous CUDA tensor of {want}")
        if src.numel() % sper:
            raise FftError(-6, f"Mdct: input holds {src.numel()} elements, expected batch * {sper}")
        batch = src.numel() // sper
        if dst is None:
            shape = (batch, self._frames, self._len) if kind == "forward" else (batch, self._signal_len)
            dst = torch.empty(shape, dtype=want, device=src.device)
        if not isinstance(dst, torch.Tensor) or dst.dtype != want or not dst.is_cuda or not dst.is_contiguous():
            raise TypeError(f"Mdct.{kind}_device wants a contiguous CUDA output tensor of {want}")
        if src.device.index != self.device or dst.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{src.device.index} / cuda:{dst.device.index}, plan is on cuda:{self.device}")
        if dst.numel() != batch * dper:
            raise FftError(-6, f"Mdct: output holds {dst.numel()} elements, expected {batch} * {dper}")
        coef = dst if kind == "forward" else src
        if self._pairs and coef.data_ptr() % (2 * coef.element_size()):
            raise TypeError(f"Mdct.{kind}_device: this plan moves coefficient pairs, so the coefficient tensor must start at an even element")
        self._lib.check(getattr(self._lib.c, f"b200fft_mdct_{kind}_device")(self._h, src.data_ptr(), dst.data_ptr(), batch,
                                                                            torch.cuda.current_stream(src.device).cuda_stream))
        return dst

    def forward(self, x: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Every row of `x` (batch * signal_len reals) into `out` (batch * frames * len reals; [batch][frames][len] when None)."""
        return self._host("forward", x, out, self._signal_len, self._frames * self._len)

    def inverse(self, coefs: np.ndarray, out: Optional[np.ndarray] = None) -> np.ndarray:
        """Every row of `coefs` (batch * frames * len reals) into `out` (batch * signal_len reals; [batch][signal_len] when None)."""
        return self._host("inverse", coefs, out, self._frames * self._len, self._signal_len)

    def forward_device(self, x, out=None):
        """forward on torch CUDA tensors (any shapes, contiguous)."""
        return self._device("forward", x, out, self._signal_len, self._frames * self._len)

    def inverse_device(self, coefs, out=None):
        """inverse on torch CUDA tensors (any shapes, contiguous)."""
        return self._device("inverse", coefs, out, self._frames * self._len, self._signal_len)


class DctNd:
    """One planned 2-D or 3-D DCT or DST: the same kind along each of the last len(shape()) axes of contiguous arrays of shape(),
    unnormalised, as scipy.fft.dctn / dstn(x, type, axes=the last r axes) / 2^r, so that Dct3n(Dct2n(x)) = Dst3n(Dst2n(x)) =
    Dct4n(Dct4n(x)) = Dst4n(Dst4n(x)) = prod(N_i / 2) x.  The last axis runs the 1-D plan of its length; every other axis runs one
    fused column pass for powers of two from 4 to 4096 (f64: 2048), or a transposition around the 1-D plan of its length.  When the
    last axis is a one-pass 1-D plan, device buffers must start at an even element (process_device raises TypeError otherwise).
    process(buffer) transforms a numpy array of whole images in place through the synchronous host entry point;
    process_device(x, out=None) takes torch CUDA tensors, in place when out is None, asynchronous on torch's current stream.
    Immutable and safe to call from many threads."""

    def __init__(self, lib: Library, shape, kind: DctKind, precision: int, device: int):
        self._lib, self._shape, self._kind, self._precision, self.device = lib, tuple(int(n) for n in shape), DctKind(kind), precision, device
        self._size = int(np.prod(self._shape, dtype=np.int64)) if self._shape else 0
        self._h = ctypes.c_void_p()
        dims = (ctypes.c_uint64 * max(1, len(self._shape)))(*self._shape)
        lib.check(lib.c.b200fft_dctn_plan_create(ctypes.byref(self._h), dims, len(self._shape), int(kind), precision, device))
        rows = self.describe().split(",rows=", 1)
        self._fused = len(rows) == 2 and re.match(r"\w+\{n=\d+,fused,", rows[1]) is not None

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            try:
                self._lib.c.b200fft_dctn_plan_destroy(h)
            except Exception:
                pass

    def shape(self) -> Tuple[int, ...]:
        return self._shape

    def kind(self) -> DctKind:
        return self._kind

    @property
    def dtype(self):
        return np.float32 if self._precision == F32 else np.float64

    def describe(self) -> str:
        buf = ctypes.create_string_buffer(1024)
        rc = self._lib.c.b200fft_dctn_describe(self._h, buf, len(buf))
        if rc < 0:
            self._lib.check(rc)
        return buf.value.decode()

    def _batch(self, n: int) -> int:
        if self._size == 0:
            return 0
        if n % self._size:
            raise FftError(-5, f"DctNd: buffer holds {n} samples, expected a multiple of {self._size}")
        return n // self._size

    def process(self, buffer: np.ndarray) -> np.ndarray:
        """Transform every array of `buffer` (batch * prod(shape()) reals, contiguous, writable) in place; returns it."""
        want = np.dtype(self.dtype)
        if not isinstance(buffer, np.ndarray) or buffer.dtype != want or not buffer.flags.c_contiguous or not buffer.flags.writeable:
            raise TypeError(f"DctNd.process wants a contiguous writable {want.name} array")
        batch = self._batch(buffer.size)
        self._lib.check(self._lib.c.b200fft_dctn_host(self._h, buffer.ctypes.data, buffer.ctypes.data, batch))
        return buffer

    def process_device(self, x, out=None):
        """x: torch CUDA tensor of batch * prod(shape()) reals (any shape, contiguous); in place when `out` is None.  Returns the result."""
        import torch

        want = torch.float32 if self._precision == F32 else torch.float64
        dst = x if out is None else out
        if not isinstance(dst, torch.Tensor) or x.dtype != want or dst.dtype != want or not x.is_cuda or not dst.is_cuda \
                or not x.is_contiguous() or not dst.is_contiguous():
            raise TypeError(f"DctNd.process_device wants contiguous CUDA tensors of {want}")
        if x.device.index != self.device or dst.device.index != self.device:
            raise FftError(-1, f"tensors are on cuda:{x.device.index} / cuda:{dst.device.index}, plan is on cuda:{self.device}")
        if dst.numel() != x.numel():
            raise FftError(-6, f"DctNd: input holds {x.numel()} samples, output {dst.numel()}: expected equal sizes")
        if self._fused and (x.data_ptr() | dst.data_ptr()) % (2 * x.element_size()):
            raise TypeError("DctNd.process_device: a one-pass row plan needs tensors that start at an even element (it moves element pairs)")
        batch = self._batch(x.numel())
        self._lib.check(self._lib.c.b200fft_dctn_device(self._h, x.data_ptr(), dst.data_ptr(), batch,
                                                        torch.cuda.current_stream(x.device).cuda_stream))
        return dst


class DctPlanner:
    """Plans Dct instances, cached per (kind, length) like rustdct's DctPlanner over rustfft's FftPlanner, and DctNd instances
    (plan_nd), cached per (kind, shape)."""

    def __init__(self, dtype=np.float32, device: int = 0, lib: Optional[Library] = None):
        dt = np.dtype(dtype)
        if dt == np.dtype(np.float32):
            self._precision = F32
        elif dt == np.dtype(np.float64):
            self._precision = F64
        else:
            raise TypeError("DctPlanner accelerates f32 and f64 only")
        self._lib = lib if lib is not None else default_library()
        if self._lib.device_count() <= 0:
            raise FftError(-2, "no sm_90 CUDA device is visible (there is no CPU fallback)")
        self.device = device
        self._cache: Dict[Tuple[int, int], Dct] = {}
        self._cache_nd: Dict[Tuple[int, Tuple[int, ...]], DctNd] = {}
        self._cache_mdct: Dict[Tuple[int, bytes, int], Mdct] = {}
        self._lock = threading.Lock()

    def plan(self, kind: DctKind, len: int) -> Dct:
        key = (int(kind), int(len))
        with self._lock:
            d = self._cache.get(key)
            if d is None:
                d = self._cache[key] = Dct(self._lib, key[1], DctKind(kind), self._precision, self.device)
            return d

    def plan_nd(self, kind: DctKind, shape) -> DctNd:
        """The same kind along each of the last len(shape) (2 or 3) axes of contiguous arrays of `shape`."""
        key = (int(kind), tuple(int(n) for n in shape))
        with self._lock:
            d = self._cache_nd.get(key)
            if d is None:
                d = self._cache_nd[key] = DctNd(self._lib, key[1], DctKind(kind), self._precision, self.device)
            return d

    def plan_dct2(self, len: int) -> Dct:
        return self.plan(DctKind.Dct2, len)

    def plan_dct3(self, len: int) -> Dct:
        return self.plan(DctKind.Dct3, len)

    def plan_dct4(self, len: int) -> Dct:
        return self.plan(DctKind.Dct4, len)

    def plan_dst2(self, len: int) -> Dct:
        return self.plan(DctKind.Dst2, len)

    def plan_dst3(self, len: int) -> Dct:
        return self.plan(DctKind.Dst3, len)

    def plan_dst4(self, len: int) -> Dct:
        return self.plan(DctKind.Dst4, len)

    def plan_mdct(self, len: int, window, signal_len: int) -> Mdct:
        """The MDCT of `len` (even) coefficients per frame over rows of signal_len samples; `window` is an array of 2 * len taps or
        "sine" / "vorbis" (rustdct's window_fn).  Cached per (len, window values, signal_len); see Mdct."""
        dt = np.float32 if self._precision == F32 else np.float64
        if isinstance(window, str):
            w = mdct_window(window, max(int(len), 0), dt)
        else:
            if np.iscomplexobj(window):
                raise TypeError("an MDCT plan needs a real window")
            w = np.ascontiguousarray(np.asarray(window), dtype=dt)
            if w.ndim != 1 or w.size != 2 * int(len):
                raise FftError(-1, f"an MDCT of len {int(len)} needs a 1-D window of {2 * int(len)} taps (got shape {w.shape})")
        key = (int(len), w.tobytes(), int(signal_len))
        with self._lock:
            m = self._cache_mdct.get(key)
            if m is None:
                m = self._cache_mdct[key] = Mdct(self._lib, key[0], w, key[2], self._precision, self.device)
            return m


def shard_range(batch: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous batch shard [lo, hi) of `rank` (remainder to the low ranks): transforms in a
    batch are independent (src/array_utils.rs:164-170 is a plain loop), so a batch shards across
    GPUs with no data-path collective."""
    base, rem = divmod(batch, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)
