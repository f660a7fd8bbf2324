"""ctypes/numpy front-end of the CPU oracle (oracle/gs_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of gs_oracle.c.  Imported only by
tests/, __graft_entry__.smoke() and bench.py (cpu_baseline / --impl reference).
PARITY UNPINNED: the reference ships no golden vectors for this path and its
rasterizer source is absent (SURVEY.md section 0); the oracle is pinned by
hand-derived known answers, fp64 finite differences and an independent autograd
restatement (tests/test_oracle_*.py).

The argument names mirror the reference call site
(PF3plat's src/model/decoder/cuda_splatting.py:99-124).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from dataclasses import dataclass

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIBS: dict[str, ctypes.CDLL] = {}


def build() -> None:
    """Compile the two oracle libraries (gcc only; a few seconds)."""
    subprocess.run(["make", "-s", "-C", _HERE], check=True)


def set_threads(n: int) -> int:
    """Sets the OpenMP thread count of both oracle libraries; returns the count in effect (1 without OpenMP)."""
    return min(int(_lib(d).gso_set_threads(int(n))) for d in (np.float32, np.float64))


def set_depth_tie_ulps(ulps: float) -> None:
    """Fragility flags only: width (in fp32 ulps) of the "undecided depth order" band; 0 disables it (see gs_oracle.c)."""
    for d in (np.float32, np.float64):
        _lib(d).gso_set_depth_tie_ulps(ctypes.c_float(ulps))


def _lib(dtype) -> ctypes.CDLL:
    name = "f64" if np.dtype(dtype) == np.float64 else "f32"
    if name not in _LIBS:
        path = os.path.join(_HERE, f"libgs_oracle_{name}.so")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "gs_oracle.c")):
            build()
        lib = ctypes.CDLL(path)
        lib.gso_forward.restype = ctypes.c_void_p
        lib.gso_forward.argtypes = [ctypes.c_void_p] * 11 + [ctypes.c_double]
        lib.gso_backward.restype = None
        lib.gso_backward.argtypes = [ctypes.c_void_p] * 11
        lib.gso_free.argtypes = [ctypes.c_void_p]
        lib.gso_set_threads.restype = ctypes.c_int
        lib.gso_set_threads.argtypes = [ctypes.c_int]
        lib.gso_set_depth_tie_ulps.restype = None
        lib.gso_set_depth_tie_ulps.argtypes = [ctypes.c_float]
        for f in ("gso_num_rendered", "gso_num_visible", "gso_num_pairs"):
            getattr(lib, f).restype = ctypes.c_int64
            getattr(lib, f).argtypes = [ctypes.c_void_p]
        for f in ("gso_depths", "gso_xy", "gso_conic_opacity", "gso_rgb", "gso_final_T", "gso_n_contrib",
                  "gso_tiles_touched", "gso_point_list", "gso_ranges", "gso_px_fragile", "gso_geom_fragile",
                  "gso_clamped"):
            getattr(lib, f).restype = ctypes.c_void_p
            getattr(lib, f).argtypes = [ctypes.c_void_p]
        _LIBS[name] = lib
    return _LIBS[name]


def _params_struct(real):
    class Params(ctypes.Structure):
        _fields_ = [
            ("P", ctypes.c_int32), ("M", ctypes.c_int32), ("sh_degree", ctypes.c_int32),
            ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("prefiltered", ctypes.c_int32),
            ("sh_eval_max_degree", ctypes.c_int32), ("pad_", ctypes.c_int32),
            ("tanfovx", real), ("tanfovy", real), ("scale_modifier", real),
            ("near_cull_z", real), ("dilation", real), ("guard_band", real),
            ("bg", real * 3), ("view", real * 16), ("proj", real * 16), ("campos", real * 3),
        ]
    return Params


@dataclass
class OracleSettings:
    """Same twelve fields as GaussianRasterizationSettings (cuda_splatting.py:99-112);
    matrices are the TRANSPOSED (row-vector convention) 4x4s exactly as the call site passes them."""
    image_height: int
    image_width: int
    tanfovx: float
    tanfovy: float
    bg: np.ndarray
    scale_modifier: float
    viewmatrix: np.ndarray
    projmatrix: np.ndarray
    sh_degree: int
    campos: np.ndarray
    prefiltered: bool = False
    debug: bool = False
    # named constants of the upstream algorithm (SURVEY.md Appendix C.1)
    near_cull_z: float = 0.2
    dilation: float = 0.3
    guard_band: float = 1.3
    sh_eval_max_degree: int = 3


def _arr(x, dtype, shape=None):
    if x is None:
        return None
    a = np.ascontiguousarray(np.asarray(x, dtype=dtype))
    if shape is not None:
        a = a.reshape(shape)
    return a


def _ptr(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


class OracleRender:
    """One forward render; holds the saved state for `backward` and exposes the intermediates."""

    def __init__(self, settings: OracleSettings, means3D, opacities, shs=None, colors_precomp=None, scales=None,
                 rotations=None, cov3D_precomp=None, dtype=np.float32, with_depth=False, frag_rel=1e-4):
        if (shs is None) == (colors_precomp is None):
            raise ValueError("Please provide excatly one of either SHs or precomputed colors!")
        if ((scales is None or rotations is None) and cov3D_precomp is None) or (
                (scales is not None or rotations is not None) and cov3D_precomp is not None):
            raise ValueError("Please provide exactly one of either scale/rotation pair or precomputed 3D covariance!")
        self.dtype = np.dtype(dtype)
        self.lib = _lib(dtype)
        real = ctypes.c_double if self.dtype == np.float64 else ctypes.c_float
        s = settings
        means3D = _arr(means3D, dtype)
        P = means3D.shape[0]
        self.P, self.H, self.W = P, int(s.image_height), int(s.image_width)
        shs = _arr(shs, dtype)
        self.M = 0 if shs is None else shs.shape[1]
        prm = _params_struct(real)()
        prm.P, prm.M, prm.sh_degree, prm.H, prm.W = P, self.M, int(s.sh_degree), self.H, self.W
        prm.prefiltered = int(s.prefiltered)
        prm.sh_eval_max_degree = int(s.sh_eval_max_degree)
        prm.tanfovx, prm.tanfovy, prm.scale_modifier = float(s.tanfovx), float(s.tanfovy), float(s.scale_modifier)
        prm.near_cull_z, prm.dilation, prm.guard_band = s.near_cull_z, s.dilation, s.guard_band
        prm.bg[:] = [float(v) for v in np.asarray(s.bg).reshape(3)]
        prm.view[:] = [float(v) for v in np.asarray(s.viewmatrix).reshape(16)]
        prm.proj[:] = [float(v) for v in np.asarray(s.projmatrix).reshape(16)]
        prm.campos[:] = [float(v) for v in np.asarray(s.campos).reshape(3)]
        self._keep = [means3D, shs, _arr(colors_precomp, dtype), _arr(opacities, dtype, (P,)), _arr(scales, dtype),
                      _arr(rotations, dtype), _arr(cov3D_precomp, dtype)]
        self.color = np.zeros((3, self.H, self.W), dtype)
        self.depth = np.zeros((self.H, self.W), dtype) if with_depth else None
        self.radii = np.zeros((P,), np.int32)
        self.handle = self.lib.gso_forward(ctypes.byref(prm), *[_ptr(a) for a in self._keep], _ptr(self.color),
                                           _ptr(self.depth), _ptr(self.radii), float(frag_rel))
        self.num_rendered = int(self.lib.gso_num_rendered(self.handle))
        self.num_visible = int(self.lib.gso_num_visible(self.handle))
        self.num_pairs = int(self.lib.gso_num_pairs(self.handle))
        self.has_sh = shs is not None
        self.has_scales = scales is not None
        # what the SH colour was evaluated from: lets a test recompute the value the clamp at 0 saw
        self.means3D, self.shs = means3D, shs
        self.campos = np.asarray(s.campos, np.float64).reshape(3)
        self.sh_eval_degree = min(int(s.sh_degree), int(s.sh_eval_max_degree))

    def _view(self, fn, dtype, shape):
        p = getattr(self.lib, fn)(self.handle)
        n = int(np.prod(shape))
        if n == 0:
            return np.zeros(shape, dtype)
        buf = (ctypes.c_char * (n * np.dtype(dtype).itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=dtype).reshape(shape).copy()

    @property
    def depths(self): return self._view("gso_depths", self.dtype, (self.P,))
    @property
    def xy(self): return self._view("gso_xy", self.dtype, (self.P, 2))
    @property
    def conic_opacity(self): return self._view("gso_conic_opacity", self.dtype, (self.P, 4))
    @property
    def rgb(self): return self._view("gso_rgb", self.dtype, (self.P, 3))
    @property
    def final_T(self): return self._view("gso_final_T", self.dtype, (self.H, self.W))
    @property
    def n_contrib(self): return self._view("gso_n_contrib", np.int32, (self.H, self.W))
    @property
    def tiles_touched(self): return self._view("gso_tiles_touched", np.int32, (self.P,))
    @property
    def point_list(self): return self._view("gso_point_list", np.uint32, (self.num_rendered,))
    @property
    def ranges(self):
        nt = ((self.W + 15) // 16) * ((self.H + 15) // 16)
        return self._view("gso_ranges", np.int64, (nt, 2))
    @property
    def px_fragile(self): return self._view("gso_px_fragile", np.uint8, (self.H, self.W)).astype(bool)
    @property
    def geom_fragile(self): return self._view("gso_geom_fragile", np.uint8, (self.P,)).astype(bool)
    @property
    def geom_fragile_bits(self): return self._view("gso_geom_fragile", np.uint8, (self.P,))   # 1 radius, 2 cull, 4 rect
    @property
    def clamped(self): return self._view("gso_clamped", np.uint8, (self.P, 3)).astype(bool)

    def backward(self, dL_dcolor, dL_ddepth=None) -> dict:
        """Returns the gradients the reference's autograd Function returns (SURVEY.md section 8 a3)."""
        P, M, dt = self.P, self.M, self.dtype
        g = {
            "means3D": np.zeros((P, 3), dt), "means2D": np.zeros((P, 3), dt),
            "shs": np.zeros((P, M, 3), dt) if self.has_sh else None,
            "colors_precomp": None if self.has_sh else np.zeros((P, 3), dt),
            "opacities": np.zeros((P, 1), dt),
            "scales": np.zeros((P, 3), dt) if self.has_scales else None,
            "rotations": np.zeros((P, 4), dt) if self.has_scales else None,
            "cov3D_precomp": None if self.has_scales else np.zeros((P, 6), dt),
        }
        dLc = _arr(dL_dcolor, dt, (3, self.H, self.W))
        dLd = _arr(dL_ddepth, dt, (self.H, self.W)) if dL_ddepth is not None else None
        self.lib.gso_backward(self.handle, _ptr(dLc), _ptr(dLd), _ptr(g["means3D"]), _ptr(g["means2D"]),
                              _ptr(g["shs"]), _ptr(g["colors_precomp"]), _ptr(g["opacities"]), _ptr(g["scales"]),
                              _ptr(g["rotations"]), _ptr(g["cov3D_precomp"]))
        return g

    def close(self):
        if self.handle:
            self.lib.gso_free(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
