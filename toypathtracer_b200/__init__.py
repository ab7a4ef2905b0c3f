"""toypathtracer_b200 — host-side mirror of the reference's renderer API (Cpp/Source/Test.h:10-17) on top of
the H100 (sm_90a) CUDA library (include/tpt_b200.h).

Two layers, both thin ctypes bindings over in-tree shared libraries built by `csrc/Makefile`:

* the six functions of the reference's ``Test.h`` — ``InitializeTest, ShutdownTest, UpdateTest, DrawTest,
  GetObjectCount, GetSceneDesc`` — bound to the *C++-mangled* symbols of ``libtoytest_b200.so``, i.e. exactly
  what a reference shell (Cpp/Windows/TestWin.cpp:76,258,265,315-316) would link against;
* :class:`Context`, the C-ABI itself (``tpt_create/tpt_set_scene/tpt_draw/...``) for runtime scenes, frame
  batching, row sharding across GPUs and device-resident buffers.

There is no CPU rendering path: importing works anywhere (so that CPU-only tests can check symbols), but any
draw without the compiled library or without a CUDA device raises.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional, Sequence, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("TPT_LIB_PATH") or os.path.join(_HERE, "libtpt_b200.so")   # override: A/B builds in experiments
SHIM_PATH = os.path.join(_HERE, "libtoytest_b200.so")

MODE_EXACT = 0
MODE_FAST = 1
MODE_REFGPU = 2        # the reference's GPU-shader estimator (ComputeShader.hlsl), strict arithmetic
MODE_REFGPU_FAST = 3   # the same with GPU-native arithmetic
kFlagAnimate = 1      # Cpp/Source/Test.h:6
kFlagProgressive = 2  # Cpp/Source/Test.h:7

SPHERE_DTYPE = np.dtype([("center", np.float32, 3), ("radius", np.float32), ("invRadius", np.float32)])  # 20 B, Maths.h:354-364
MATERIAL_DTYPE = np.dtype([("type", np.int32), ("albedo", np.float32, 3), ("emissive", np.float32, 3),
                           ("roughness", np.float32), ("ri", np.float32)])                                # 36 B, Test.cpp:36-44
CAMERA_DTYPE = np.dtype([("origin", np.float32, 3), ("lowerLeftCorner", np.float32, 3), ("horizontal", np.float32, 3),
                         ("vertical", np.float32, 3), ("uu", np.float32, 3), ("vv", np.float32, 3), ("ww", np.float32, 3),
                         ("lensRadius", np.float32)])                                                     # 88 B, Maths.h:444-449
assert SPHERE_DTYPE.itemsize == 20 and MATERIAL_DTYPE.itemsize == 36 and CAMERA_DTYPE.itemsize == 88


class TptError(RuntimeError):
    pass


_lib = None
_shim = None


def _load_lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise TptError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(or `make -C toypathtracer_b200/csrc`). There is no CPU fallback.")
    L = ctypes.CDLL(LIB_PATH, mode=ctypes.RTLD_GLOBAL)
    vp, ci, cu, cll = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint, ctypes.c_longlong
    L.tpt_create.argtypes = [ci, ctypes.POINTER(vp)]; L.tpt_create.restype = ci
    L.tpt_destroy.argtypes = [vp]; L.tpt_destroy.restype = None
    L.tpt_device_count.argtypes = []; L.tpt_device_count.restype = ci
    L.tpt_last_error.argtypes = [vp]; L.tpt_last_error.restype = ctypes.c_char_p
    L.tpt_set_scene.argtypes = [vp, vp, vp, ci, vp, vp, ci]; L.tpt_set_scene.restype = ci
    L.tpt_set_camera.argtypes = [vp, vp]; L.tpt_set_camera.restype = ci
    L.tpt_set_spp.argtypes = [vp, ci]; L.tpt_set_spp.restype = ci
    L.tpt_set_option.argtypes = [vp, ctypes.c_char_p, ci]; L.tpt_set_option.restype = ci
    L.tpt_draw.argtypes = [vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, ci, cu, ci, ctypes.POINTER(cll), ctypes.POINTER(cll), vp]
    L.tpt_draw.restype = ci
    L.tpt_read_ray_count.argtypes = [vp, vp, ctypes.POINTER(cll)]; L.tpt_read_ray_count.restype = ci
    L.tpt_last_kernel_ms.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]; L.tpt_last_kernel_ms.restype = ci
    L.tpt_last_launch_count.argtypes = [vp]; L.tpt_last_launch_count.restype = ci
    L.tpt_last_scene_upload_bytes.argtypes = [vp]; L.tpt_last_scene_upload_bytes.restype = ctypes.c_longlong
    L.tpt_tonemap_srgb8.argtypes = [vp, vp, ci, ci, ci, vp, ci, vp]; L.tpt_tonemap_srgb8.restype = ci
    L.tpt_tonemap_rgba8.argtypes = [vp, vp, ci, ci, ci, vp, ci, ci, ci, ci, vp]; L.tpt_tonemap_rgba8.restype = ci
    L.tpt_debug_libm.argtypes = [vp, ci, vp, vp, cll]; L.tpt_debug_libm.restype = ci
    L.tpt_debug_hit.argtypes = [vp, ci, vp, vp, vp, cll]; L.tpt_debug_hit.restype = ci
    L.tpt_debug_last_kernels.argtypes = [vp, ctypes.c_char_p, ci]; L.tpt_debug_last_kernels.restype = ci
    L.tpt_trace_rays.argtypes = [vp, vp, ci, cll, ci, ci, vp, ci, ctypes.POINTER(cll), vp]; L.tpt_trace_rays.restype = ci
    L.tpt_trace_irradiance.argtypes = [vp, vp, vp, ci, cll, ci, ci, vp, ci, ctypes.POINTER(cll), vp]
    L.tpt_trace_irradiance.restype = ci
    L.tpt_draw_aovs.argtypes = [vp, ci, ci, ci, ci, ci, ci, ci, ci, vp, vp, vp, ci, cu, ctypes.POINTER(cll), vp]
    L.tpt_draw_aovs.restype = ci
    L.tpt_trace_aovs.argtypes = [vp, vp, ci, cll, vp, vp, vp, ci, ctypes.POINTER(cll), vp]; L.tpt_trace_aovs.restype = ci
    L.tpt_draw_samples.argtypes = [vp, ci, ci, ci, vp, cll, ci, vp, vp, ci, ctypes.POINTER(cll), vp]
    L.tpt_draw_samples.restype = ci
    L.tpt_trace_samples.argtypes = [vp, vp, vp, ci, cll, vp, cll, ci, ci, vp, vp, ci, ctypes.POINTER(cll), vp]
    L.tpt_trace_samples.restype = ci
    L.tpt_set_environment.argtypes = [vp, vp, ci, ci, ci]; L.tpt_set_environment.restype = ci
    L.tpt_set_textures.argtypes = [vp, vp, ci, ci, ci, vp, ci, ci]; L.tpt_set_textures.restype = ci
    L.tpt_set_emission_textures.argtypes = [vp, vp, ci, ci, ci, vp, ci, ci]; L.tpt_set_emission_textures.restype = ci
    L.tpt_set_media.argtypes = [vp, vp, ci]; L.tpt_set_media.restype = ci
    L.tpt_set_fog.argtypes = [vp, vp]; L.tpt_set_fog.restype = ci
    cull = ctypes.c_ulonglong
    L.tpt_mem_alloc.argtypes = [vp, cull, ctypes.POINTER(vp)]; L.tpt_mem_alloc.restype = ci
    L.tpt_mem_free.argtypes = [vp, vp]; L.tpt_mem_free.restype = ci
    L.tpt_mem_copy.argtypes = [vp, vp, vp, cull, ci]; L.tpt_mem_copy.restype = ci
    L.tpt_ipc_export.argtypes = [vp, vp, vp]; L.tpt_ipc_export.restype = ci
    L.tpt_ipc_open.argtypes = [vp, vp, ctypes.POINTER(vp)]; L.tpt_ipc_open.restype = ci
    L.tpt_ipc_close.argtypes = [vp, vp]; L.tpt_ipc_close.restype = ci
    _lib = L
    return L


def device_count() -> int:
    return int(_load_lib().tpt_device_count())


class DevicePtr:
    """A raw device address (e.g. an image living in another rank's HBM, opened with Context.ipc_open)."""

    def __init__(self, addr: int):
        self.addr = int(addr)


def _as_ptr(buf, dtype: str = "float32") -> Tuple[int, bool, object]:
    """(address, on_device, keepalive) for a numpy array, a torch tensor or a raw device address of element type `dtype`
    ("float32", or "int32" for id buffers)."""
    if isinstance(buf, DevicePtr):
        return buf.addr, True, buf
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.dtype(dtype) or not buf.flags["C_CONTIGUOUS"]:
            raise TptError(f"backbuffer must be a C-contiguous {dtype} array")
        return buf.ctypes.data, False, buf
    if hasattr(buf, "data_ptr"):  # torch tensor
        if not buf.is_contiguous() or str(buf.dtype) != f"torch.{dtype}":
            raise TptError(f"backbuffer tensor must be contiguous {dtype}")
        return int(buf.data_ptr()), bool(buf.is_cuda), buf
    raise TptError("unsupported backbuffer type")


def _numel(buf) -> int:
    return int(buf.size) if isinstance(buf, np.ndarray) else int(buf.numel())


_CUDA_STREAM_LEGACY = 1            # cudaStreamLegacy: torch's default stream, whose handle reads as 0
_NO_ENTRIES = (ctypes.c_int * 1)()  # the address passed for an empty buffer: it has no data pointer, and NULL means "none"


def _entries(what: str, name: str, buf, n, row: Tuple[int, ...]) -> int:
    """The entry count of a caller input `name` of shape (N, *row), or of a DevicePtr, which needs `n`; a given n must
    match the buffer."""
    if isinstance(buf, DevicePtr):
        if n is None:
            raise TptError(f"{what}: a DevicePtr needs n")
        return int(n)
    if tuple(buf.shape[1:]) != row or len(buf.shape) != 1 + len(row):
        raise TptError(f"{what}: {name} must have shape (N,{''.join(f' {d}' for d in row)})")
    if n is not None and int(n) != buf.shape[0]:
        raise TptError(f"{what}: n does not match {name}")
    return int(buf.shape[0])


def _buffer_ptrs(what: str, bufs, entries: int):
    """Addresses of the given buffers among `bufs`, (name, buffer or None, dtype, values per entry) each, which must hold
    `entries` entries unless a DevicePtr; their common kind (on device or not) and keepalives."""
    ptrs, kinds, keep = [], set(), []
    for name, buf, dtype, per in bufs:
        if buf is None:
            ptrs.append(None)
            continue
        if not isinstance(buf, DevicePtr) and _numel(buf) != entries * per:
            raise TptError(f"{what}: {name} must hold {entries} x {per} {dtype} values, not {_numel(buf)}")
        addr, on_dev, k = _as_ptr(buf, dtype)
        if addr == 0 and entries == 0:
            addr = ctypes.addressof(_NO_ENTRIES)
        ptrs.append(ctypes.c_void_p(addr)); kinds.add(on_dev); keep.append(k)
    names = [b[0] for b in bufs]
    if not kinds:
        raise TptError(f"{what}: no output buffer ({', '.join(names[:-1])} or {names[-1]})")
    if len(kinds) > 1:
        raise TptError(f"{what}: {', '.join(names[:-1])} and {names[-1]} must be all host or all device buffers")
    return ptrs, kinds.pop(), keep


def _aovs(albedo, normal, ids):
    """The AOV outputs for _buffer_ptrs: float4 albedo and normal, int32 ids."""
    return [("albedo", albedo, "float32", 4), ("normal", normal, "float32", 4), ("ids", ids, "int32", 1)]


def _alloc_like(like, device: int, specs):
    """New outputs of (shape, dtype name) `specs` of the kind of input `like`: numpy arrays for a numpy array, else torch
    tensors on like's device (CUDA device `device` for a DevicePtr)."""
    if isinstance(like, np.ndarray):
        return [np.empty(shape, dtype) for shape, dtype in specs]
    import torch
    dev = like.device if hasattr(like, "device") else torch.device("cuda", device)
    return [torch.empty(shape, dtype=getattr(torch, dtype), device=dev) for shape, dtype in specs]


def _cuda_device(*bufs):
    """The device of the first CUDA torch tensor among bufs, or None."""
    for b in bufs:
        if getattr(b, "is_cuda", False):
            return b.device
    return None


def _torch_stream(dev) -> int:
    """Handle of torch's current stream on `dev` for the library's cudaStream argument (0 would mean the context's own
    stream, so torch's legacy default stream is passed as cudaStreamLegacy)."""
    import torch
    return torch.cuda.current_stream(dev).cuda_stream or _CUDA_STREAM_LEGACY


def kernel_signature(mangled: str) -> str:
    """A kernel's mangled name as its template instance, the namespace and parameter list dropped:
    '_ZN3tpt12k_fast_queueILi128ELi6ELi4EEEv...' -> 'k_fast_queue<128, 6, 4>', '_ZN3tpt8k_refgpuILb0ENS_9RgSetupK2EEEv...'
    -> 'k_refgpu<false, RgSetupK2>'. Decodes the part of the Itanium C++ ABI mangling the library's kernels use (nested
    names, substitutions, integer and bool literals, class template arguments), so no demangler is needed."""
    s = mangled
    if not s.startswith("_Z"):
        return s
    pos = 2

    def source():                       # <length><identifier>
        nonlocal pos
        i = pos
        while s[pos].isdigit():
            pos += 1
        n = int(s[i:pos])
        pos += n
        return s[pos - n:pos]

    def targs():                        # I <arg>+ E
        nonlocal pos
        pos += 1
        out = []
        while s[pos] != "E":
            if s[pos] == "L":           # L <type> <value> E
                t = s[pos + 1]
                j = s.index("E", pos)
                v = s[pos + 2:j]
                pos = j + 1
                out.append(("true" if v == "1" else "false") if t == "b" else ("-" + v[1:] if v.startswith("n") else v))
            else:
                out.append(name())
        pos += 1
        return "<" + ", ".join(out) + ">"

    def name():
        nonlocal pos
        nested = s[pos] == "N"
        if nested:
            pos += 1
        out = ""
        while True:
            c = s[pos]
            if c == "I":
                out += targs()
            elif c == "S":              # a substitution (here: the namespace seen before)
                pos = s.index("_", pos) + 1
            elif c.isdigit():
                part = source()
                if part != "tpt":
                    out += ("::" if out else "") + part
            else:
                break
            if not nested and s[pos] != "I":
                break
        if nested:
            pos += 1                    # E
        return out

    return name()


LUMA = (0.2126, 0.7152, 0.0722)    # Rec. 709 luminance weights of the adaptive stopping rule


def adaptive_pixels(sum4, sq4, rel_err: float, max_spp: int, shape: Optional[Tuple[int, int]] = None):
    """The stopping rule of Context.render_adaptive, on torch tensors of draw_samples sums (N, 4) and squares (N, 4):
    the int32 indices of the pixels that have fewer than max_spp samples and whose standard error of the mean luminance
    exceeds rel_err * (mean luminance + 0.05). Per channel the variance is the unbiased sample variance
    (sq - sum^2 / n) / (n - 1); the moments hold no covariances between channels, so the luminance's standard error is
    taken as sum_c LUMA_c * se_c, an upper bound that is exact when the channels' noise is fully correlated (a path's
    colour mostly scales as one). A pixel with one sample has no variance estimate and is always picked.
    With shape = (height, width) (the sums of a whole image, row-major) the picked set is grown by the 3 x 3
    neighbourhood of every picked pixel. A few samples cannot see a rare event: a pixel on the edge of a light's mirror
    image whose first 4 samples all hit (or all missed) the light has a zero sample variance and would stop with a
    wrong value; its neighbours across the edge are noisy, and the dilation refines it with them."""
    import torch
    cnt = sum4[:, 3]
    n = cnt.clamp(min=2.0).unsqueeze(1)
    mean = sum4[:, :3] / n
    var = ((sq4[:, :3] - sum4[:, :3] * mean) / (n - 1.0)).clamp(min=0.0)
    w = torch.tensor(LUMA, dtype=sum4.dtype, device=sum4.device)
    se = (var / n).sqrt() @ w
    lum = (sum4[:, :3] / cnt.clamp(min=1.0).unsqueeze(1)) @ w
    noisy = (se > rel_err * (lum + 0.05)) | (cnt < 2)
    if shape is not None:
        grown = torch.nn.functional.max_pool2d(noisy.view(1, 1, *shape).to(torch.float32), 3, stride=1, padding=1)
        noisy = grown.view(-1) > 0
    return ((cnt < max_spp) & noisy).nonzero().squeeze(1).to(torch.int32)


class Context:
    """One CUDA device's renderer state (scene blob, scratch, counters): ``tpt_context`` of include/tpt_b200.h."""

    def __init__(self, device: int = 0):
        self._L = _load_lib()
        h = ctypes.c_void_p()
        rc = self._L.tpt_create(device, ctypes.byref(h))
        if rc != 0 or not h.value:
            raise TptError(f"tpt_create(device={device}) failed with CUDA error {rc}: no usable CUDA device "
                           "(this package has no CPU path)")
        self._h = h
        self.device = device
        self.count = 0
        self.spp = 4          # the library's default, kept in step by set_spp

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self._L.tpt_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc: int, what: str):
        if rc != 0:
            raise TptError(f"{what} failed ({rc}): {self._L.tpt_last_error(self._h).decode()}")

    def _call(self, fn: str, want_rays: bool, stream: int, *args) -> int:
        """Library call `fn`(context, *args, outRayCount, cudaStream) of a caller-buffer function; returns the rays it
        traced (0 when not want_rays). Stream 0 is the context's own stream."""
        total = ctypes.c_longlong(0)
        rc = getattr(self._L, fn)(self._h, *args, ctypes.byref(total) if want_rays else None,
                                  ctypes.c_void_p(stream) if stream else None)
        self._check(rc, fn)
        return int(total.value)

    def set_scene(self, spheres: np.ndarray, materials: np.ndarray, camera: np.ndarray,
                  emissives: Optional[np.ndarray] = None):
        """Raw scene as exported by GetSceneDesc (Test.cpp:377-384)."""
        spheres = np.ascontiguousarray(spheres); materials = np.ascontiguousarray(materials)
        camera = np.ascontiguousarray(camera)
        n = spheres.nbytes // 20
        if spheres.nbytes != n * 20 or materials.nbytes != n * 36 or camera.nbytes != 88:
            raise TptError("scene arrays must be n*20 B spheres, n*36 B materials, 88 B camera")
        if emissives is not None:
            emissives = np.ascontiguousarray(emissives, dtype=np.int32)
            ep, ec = emissives.ctypes.data, int(emissives.size)
        else:
            ep, ec = None, 0
        self._check(self._L.tpt_set_scene(self._h, spheres.ctypes.data, materials.ctypes.data, n,
                                          camera.ctypes.data, ep, ec), "tpt_set_scene")
        self.count = n

    def set_environment(self, image):
        """tpt_set_environment: light the fast mode with a lat-long radiance map instead of the sky. `image` is an
        (H, W, 3) or (H, W, 4) float32 numpy array or torch tensor (CPU, or CUDA on the context's device), row 0 at the
        zenith (an HDR image loaded top row first is upright), the centre column along -z; RGB is padded to RGBA and
        alpha is ignored. None removes the environment. Refused here: other shapes and dtypes, and negative (-0
        included) or non-finite RGB values. The texels are copied, and a CUDA tensor is read after torch's current stream has
        finished writing it. See include/tpt_b200.h for the mapping and which calls use the map."""
        if image is None:
            self._check(self._L.tpt_set_environment(self._h, None, 0, 0, 0), "tpt_set_environment")
            return
        if not isinstance(image, np.ndarray) and not hasattr(image, "data_ptr"):
            raise TptError("set_environment: image must be a numpy array or a torch tensor")
        shape = tuple(image.shape)
        if len(shape) != 3 or shape[2] not in (3, 4):
            raise TptError(f"set_environment: image must have shape (H, W, 3) or (H, W, 4), not {shape}")
        if isinstance(image, np.ndarray):
            if image.dtype != np.float32:
                raise TptError(f"set_environment: image must be float32, not {image.dtype}")
            rgb = image[..., :3]
            if not np.isfinite(rgb).all() or np.signbit(rgb).any():
                raise TptError("set_environment: RGB values must be finite and not negative (-0 included)")
            rgba = np.zeros(shape[:2] + (4,), np.float32)
            rgba[..., :shape[2]] = image
            addr, on_dev = rgba.ctypes.data, False
        else:
            import torch
            if image.dtype != torch.float32:
                raise TptError(f"set_environment: image must be float32, not {image.dtype}")
            rgb = image[..., :3]
            if not bool(torch.isfinite(rgb).all()) or bool(torch.signbit(rgb).any()):
                raise TptError("set_environment: RGB values must be finite and not negative (-0 included)")
            rgba = torch.zeros(shape[:2] + (4,), dtype=torch.float32, device=image.device)
            rgba[..., :shape[2]] = image
            on_dev = bool(rgba.is_cuda)
            if on_dev:
                torch.cuda.current_stream(rgba.device).synchronize()   # the library reads it on its own stream
            addr = int(rgba.data_ptr())
        self._check(self._L.tpt_set_environment(self._h, ctypes.c_void_p(addr), shape[1], shape[0], 1 if on_dev else 0),
                    "tpt_set_environment")

    def set_textures(self, textures, sphere_layers=None):
        """tpt_set_textures: lat-long albedo textures on spheres for the fast mode. `textures` is an (L, H, W, 3) or
        (L, H, W, 4) float32 numpy array or torch tensor (CPU, or CUDA on the context's device): L layers, row 0 at each
        sphere's +y pole, the centre column along -z; RGB is padded to RGBA and alpha is ignored. `sphere_layers` is a 1-D
        integer array: entry i is the layer of sphere i, or -1 for none (spheres past its end are untextured). A hit on a
        textured sphere uses albedo x the layer's lookup at its normal. None removes the textures. Refused here: other
        shapes and dtypes, negative (-0 included) or non-finite RGB values, and layers outside [-1, L). See
        include/tpt_b200.h for which calls and kernels use them."""
        self._set_texture_set("set_textures", textures, sphere_layers)

    def set_emission_textures(self, textures, sphere_layers=None):
        """tpt_set_emission_textures: lat-long emission textures on spheres for the fast mode, independent of
        set_textures. Takes the same inputs as set_textures and refuses the same ones. The emitted radiance of a hit on
        a sphere with a layer is its material's emission x the layer's lookup at the hit's normal, also where a light
        sampling shadow ray meets the light; a sphere with zero emission stays dark. None removes the textures. See
        include/tpt_b200.h for where the estimator applies it. The option "emission_texture_sampling" (set_option)
        importance-samples the textured lights by their layers, from tables this call builds."""
        self._set_texture_set("set_emission_textures", textures, sphere_layers)

    def _set_texture_set(self, name, textures, sphere_layers):
        """set_textures and set_emission_textures (`name`): checks and stages their inputs for tpt_<name>, which is looked
        up only once they pass."""
        cname = "tpt_" + name
        if textures is None:
            self._check(getattr(self._L, cname)(self._h, None, 0, 0, 0, None, 0, 0), cname)
            return
        if not isinstance(textures, np.ndarray) and not hasattr(textures, "data_ptr"):
            raise TptError(f"{name}: textures must be a numpy array or a torch tensor")
        shape = tuple(textures.shape)
        if len(shape) != 4 or shape[3] not in (3, 4) or 0 in shape:
            raise TptError(f"{name}: textures must have shape (L, H, W, 3) or (L, H, W, 4) with L, H, W >= 1, not {shape}")
        if sphere_layers is None:
            raise TptError(f"{name}: sphere_layers is required with textures")
        layers = np.asarray(sphere_layers.cpu() if hasattr(sphere_layers, "cpu") else sphere_layers)
        if layers.ndim != 1 or layers.dtype.kind not in "iu":
            raise TptError(f"{name}: sphere_layers must be a 1-D integer array, not {layers.dtype} of shape {layers.shape}")
        bad = np.nonzero((layers < -1) | (layers >= shape[0]))[0]
        if bad.size:
            i = int(bad[0])
            raise TptError(f"{name}: sphere_layers[{i}] = {int(layers[i])} is outside [-1, {shape[0]})")
        layers = np.ascontiguousarray(layers, dtype=np.int32)
        if isinstance(textures, np.ndarray):
            if textures.dtype != np.float32:
                raise TptError(f"{name}: textures must be float32, not {textures.dtype}")
            rgb = textures[..., :3]
            if not np.isfinite(rgb).all() or np.signbit(rgb).any():
                raise TptError(f"{name}: RGB values must be finite and not negative (-0 included)")
            rgba = np.zeros(shape[:3] + (4,), np.float32)
            rgba[..., :shape[3]] = textures
            addr, on_dev = rgba.ctypes.data, False
        else:
            import torch
            if textures.dtype != torch.float32:
                raise TptError(f"{name}: textures must be float32, not {textures.dtype}")
            rgb = textures[..., :3]
            if not bool(torch.isfinite(rgb).all()) or bool(torch.signbit(rgb).any()):
                raise TptError(f"{name}: RGB values must be finite and not negative (-0 included)")
            rgba = torch.zeros(shape[:3] + (4,), dtype=torch.float32, device=textures.device)
            rgba[..., :shape[3]] = textures
            on_dev = bool(rgba.is_cuda)
            if on_dev:
                torch.cuda.current_stream(rgba.device).synchronize()   # the library reads it on its own stream
            addr = int(rgba.data_ptr())
        self._check(getattr(self._L, cname)(self._h, ctypes.c_void_p(addr), shape[2], shape[1], shape[0],
                                            layers.ctypes.data if layers.size else None, int(layers.size),
                                            1 if on_dev else 0), cname)

    def set_media(self, media):
        """tpt_set_media: homogeneous media inside glass spheres for the fast mode. `media` is an (N, 5) float32 numpy
        array or CPU torch tensor, row i {sigma_a.r, sigma_a.g, sigma_a.b, sigma_s, g} the medium inside sphere i (all
        sigmas zero: none; spheres past N have none), or None to remove all media. A medium acts only inside glass.
        Refused here, as by the library: other shapes and dtypes, a non-finite sigma or one with its sign bit set (-0
        included), a g that is NaN or has |g| >= 1. See include/tpt_b200.h for the estimator and which calls use it."""
        if media is None:
            self._check(self._L.tpt_set_media(self._h, None, 0), "tpt_set_media")
            return
        if hasattr(media, "data_ptr"):
            if media.is_cuda:
                raise TptError("set_media: media must be in host memory (a numpy array or a CPU tensor)")
            media = media.numpy()
        if not isinstance(media, np.ndarray):
            raise TptError("set_media: media must be a numpy array or a CPU torch tensor")
        if media.ndim != 2 or media.shape[1] != 5:
            raise TptError(f"set_media: media must have shape (N, 5), not {tuple(media.shape)}")
        if media.dtype != np.float32:
            raise TptError(f"set_media: media must be float32, not {media.dtype}")
        fields = ("sigma_a.r", "sigma_a.g", "sigma_a.b", "sigma_s", "g")
        for i, row in enumerate(media):
            for f in range(4):
                if not np.isfinite(row[f]) or np.signbit(row[f]):
                    raise TptError(f"set_media: sphere {i} has {fields[f]} = {float(row[f]):g}")
            if not abs(float(row[4])) < 1.0:
                raise TptError(f"set_media: sphere {i} has g = {float(row[4]):g}")
        media = np.ascontiguousarray(media)
        self._check(self._L.tpt_set_media(self._h, media.ctypes.data if media.size else None, int(media.shape[0])),
                    "tpt_set_media")

    def set_fog(self, centre, radius=None, sigma_a=None, sigma_s=None, g=0.0):
        """tpt_set_fog: homogeneous fog in the air between the spheres for the fast mode, lit by the lights. The fog fills
        the ball {centre, radius} minus the spheres; sigma_a is the absorption coefficient (a number, or one per colour
        channel), sigma_s the grey scattering coefficient and g the Henyey-Greenstein asymmetry. set_fog(None) removes it,
        as does a fog whose sigmas are all zero. Refused here, as by the library and with its field names: a non-finite
        centre, a radius that is not finite or not > 0, a sigma that is non-finite or has its sign bit set (-0 included), a
        g that is NaN or has |g| >= 1. See include/tpt_b200.h for the estimator and which calls use it."""
        if centre is None:
            self._check(self._L.tpt_set_fog(self._h, None), "tpt_set_fog")
            return
        try:
            c = np.asarray(centre, np.float64).reshape(-1)
            sa = np.asarray(sigma_a, np.float64).reshape(-1)
            rec = [float(radius), float(sigma_s), float(g)]
        except (TypeError, ValueError):
            raise TptError("set_fog: centre must be 3 numbers, and radius, sigma_a, sigma_s and g numbers") from None
        if c.size != 3:
            raise TptError(f"set_fog: centre must be 3 numbers, not {c.size}")
        if sa.size == 1:
            sa = np.repeat(sa, 3)
        if sa.size != 3:
            raise TptError(f"set_fog: sigma_a must be a number or 3 numbers, not {sa.size}")
        with np.errstate(over="ignore"):
            fog = np.array([*c, rec[0], *sa, rec[1], rec[2]], np.float32)
        names = ("centre.x", "centre.y", "centre.z", "radius", "sigma_a.r", "sigma_a.g", "sigma_a.b", "sigma_s", "g")
        for f in range(3):
            if not np.isfinite(fog[f]):
                raise TptError(f"set_fog: {names[f]} = {float(fog[f]):g}")
        if not (np.isfinite(fog[3]) and fog[3] > 0):
            raise TptError(f"set_fog: radius = {float(fog[3]):g}")
        for f in range(4, 8):
            if not np.isfinite(fog[f]) or np.signbit(fog[f]):
                raise TptError(f"set_fog: {names[f]} = {float(fog[f]):g}")
        if not abs(float(fog[8])) < 1.0:
            raise TptError(f"set_fog: g = {float(fog[8]):g}")
        self._check(self._L.tpt_set_fog(self._h, fog.ctypes.data), "tpt_set_fog")

    def set_camera(self, camera: np.ndarray):
        camera = np.ascontiguousarray(camera)
        self._check(self._L.tpt_set_camera(self._h, camera.ctypes.data), "tpt_set_camera")

    def set_spp(self, spp: int):
        self._check(self._L.tpt_set_spp(self._h, spp), "tpt_set_spp")
        self.spp = int(spp)

    def set_option(self, key: str, value: int):
        self._check(self._L.tpt_set_option(self._h, key.encode(), int(value)), f"tpt_set_option({key})")

    def draw(self, frame: int, num_frames: int, width: int, height: int, backbuffer, flags: int = 0,
             mode: int = MODE_EXACT, rows: Optional[Tuple[int, int, int, int]] = None, stream: int = 0,
             want_rays: bool = True, per_frame: bool = False):
        """tpt_draw. rows = (row0, numRows, rowStep, packed); default = the whole image.
        Returns total rays (int) if want_rays, plus the per-frame list if per_frame (exact mode)."""
        row0, nrows, step, packed = rows if rows is not None else (0, height, 1, 0)
        addr, on_dev, _keep = _as_ptr(backbuffer)
        total = ctypes.c_longlong(0)
        pf = (ctypes.c_longlong * num_frames)() if per_frame else None
        rc = self._L.tpt_draw(self._h, frame, num_frames, width, height, row0, nrows, step, packed,
                              ctypes.c_void_p(addr), 1 if on_dev else 0, flags, mode,
                              ctypes.byref(total) if want_rays else None,
                              pf if per_frame else None, ctypes.c_void_p(stream) if stream else None)
        self._check(rc, "tpt_draw")
        if per_frame:
            return int(total.value), [int(v) for v in pf]
        return int(total.value) if want_rays else None

    def trace_rays(self, rays, spp: int = 4, frame: int = 0, out=None, stream: int = 0, want_rays: bool = True, n=None):
        """tpt_trace_rays: fast-mode radiance estimates (mean of `spp` samples, streams keyed by `frame`) for caller rays
        {o.xyz, d.xyz}. `rays` is an (N, 6) float32 numpy array, a torch tensor (CPU or CUDA; a row slice is fine) or a
        DevicePtr together with `n`. Without `out` the result is a new (N, 4) array of the same kind as `rays` (numpy, CPU or
        CUDA tensor; a DevicePtr gets a CUDA tensor); `out` may be any buffer of N float4. Returns (out, rays traced), or
        out alone when want_rays is False (device buffers then stay asynchronous on `stream`)."""
        n = _entries("trace_rays", "rays", rays, n, (6,))
        raddr, ron, _keep = _as_ptr(rays)
        if out is None:
            (out,) = _alloc_like(rays, self.device, [((n, 4), "float32")])
        (po,), oon, _keep_out = _buffer_ptrs("trace_rays", [("out", out, "float32", 4)], n)
        total = self._call("tpt_trace_rays", want_rays, stream, ctypes.c_void_p(raddr), 1 if ron else 0, n, int(spp),
                           int(frame), po, 1 if oon else 0)
        return (out, total) if want_rays else out

    def trace_irradiance(self, points, ids=None, spp: int = 4, frame: int = 0, out=None, stream: int = 0,
                         want_rays: bool = True, n=None):
        """tpt_trace_irradiance: fast-mode irradiance E(p, n) (pi x the mean of `spp` samples, streams keyed by `frame`)
        at caller surface points {p.xyz, n.xyz}, in an (N, 6) float32 buffer of the kinds trace_rays takes for its rays.
        `ids` (N,) int32 of the same kind, or None: the sphere each point lies on, whose light is then not sampled from
        it; a point on an emissive sphere must pass that sphere's id. For a camera ray whose first hit is a Lambert sphere
        at (p, n), trace_rays estimates Le + albedo * E / pi. `out`, the allocation of a missing `out`, `stream` and the
        return value are as for trace_rays."""
        n = _entries("trace_irradiance", "points", points, n, (6,))
        if ids is not None:
            _entries("trace_irradiance", "ids", ids, n, ())
        (pp, pi), pon, _keep = _buffer_ptrs("trace_irradiance", [("points", points, "float32", 6), ("ids", ids, "int32", 1)], n)
        if out is None:
            (out,) = _alloc_like(points, self.device, [((n, 4), "float32")])
        (po,), oon, _keep_out = _buffer_ptrs("trace_irradiance", [("out", out, "float32", 4)], n)
        total = self._call("tpt_trace_irradiance", want_rays, stream, pp, pi, 1 if pon else 0, n, int(spp), int(frame), po,
                           1 if oon else 0)
        return (out, total) if want_rays else out

    def draw_aovs(self, frame: int, num_frames: int, width: int, height: int, albedo=None, normal=None, ids=None,
                  flags: int = 0, rows: Optional[Tuple[int, int, int, int]] = None, stream: int = 0, want_rays: bool = True):
        """tpt_draw_aovs: first-hit AOVs of the fast draw draw(frame, num_frames, width, height, ..., flags, MODE_FAST,
        rows) would make, into any of albedo (albedo.rgb, coverage), normal (normal.xyz, depth) — float32 buffers of
        4 values per pixel, blended over their contents like the image — and ids (int32, sample 0's sphere id or -1).
        Buffers hold width x height pixels (numRows with a packed row region), all host or all device; rows = (row0,
        numRows, rowStep, packed). Returns the rays traced (one per sample) if want_rays, else None."""
        row0, nrows, step, packed = rows if rows is not None else (0, height, 1, 0)
        (pa, pn, pi), on_dev, _keep = _buffer_ptrs("draw_aovs", _aovs(albedo, normal, ids), (nrows if packed else height) * width)
        total = self._call("tpt_draw_aovs", want_rays, stream, frame, num_frames, width, height, row0, nrows, step, packed,
                           pa, pn, pi, 1 if on_dev else 0, flags)
        return total if want_rays else None

    def trace_aovs(self, rays, albedo=None, normal=None, ids=None, n=None, stream: int = 0, want_rays: bool = True):
        """tpt_trace_aovs: first-hit AOVs of caller rays {o.xyz, d.xyz} (buffers as for trace_rays). albedo and normal
        receive N float4 (albedo.rgb, coverage) and (normal.xyz, depth), ids N int32 (-1: miss or untraceable ray); any
        of them may be omitted, and without all three they are allocated, (N, 4), (N, 4) and (N,), of the kind of `rays`
        (a DevicePtr gets CUDA tensors). Returns ((albedo, normal, ids), rays traced), or the tuple alone when want_rays
        is False."""
        n = _entries("trace_aovs", "rays", rays, n, (6,))
        raddr, ron, _keep = _as_ptr(rays)
        if albedo is None and normal is None and ids is None:
            albedo, normal, ids = _alloc_like(rays, self.device, [((n, 4), "float32"), ((n, 4), "float32"), (n, "int32")])
        (pa, pn, pi), oon, _keep_out = _buffer_ptrs("trace_aovs", _aovs(albedo, normal, ids), n)
        total = self._call("tpt_trace_aovs", want_rays, stream, ctypes.c_void_p(raddr), 1 if ron else 0, n, pa, pn, pi,
                           1 if oon else 0)
        return ((albedo, normal, ids), total) if want_rays else (albedo, normal, ids)

    def draw_samples(self, frame: int, width: int, height: int, pixels=None, spp: Optional[int] = None, sum4=None,
                     sq4=None, stream: int = 0, want_rays: bool = True, n=None):
        """tpt_draw_samples: `spp` more samples (default: the context's spp) of the fast draw of a width x height image for
        each entry of `pixels` — linear indices y * width + x, int32, duplicates and any order allowed; None = every
        pixel — ADDED to sum4 (sum r, g, b, sample count) and, when given, sq4 (sum r^2, g^2, b^2, 0), both (N, 4) float32.
        Sample s of pixel p at `frame` is the draw's own (stream pixel_seed(p * spp + s, frame)), so an all-pixel call at
        the context's spp traces tpt_draw(frame, 1, ..., MODE_FAST)'s samples and frames frame + 1, frame + 2, ... add
        independent ones. Buffers are numpy arrays, torch tensors (CPU or CUDA) or DevicePtr (a DevicePtr list needs
        `n`), all host or all device. Without sum4 and sq4 both are allocated zeroed, of the kind of `pixels` (a CUDA
        tensor on the context's device for pixels=None or a DevicePtr). When any buffer is a CUDA tensor (allocated ones
        included) and `stream` is 0, the call runs on torch's current stream of that device, so it is ordered with the
        torch work around it; outputs allocated for an explicit `stream` are zeroed on that stream. Returns
        ((sum4, sq4), rays traced), or the pair alone when want_rays is False. A call with a pixel list is synchronous."""
        numpix = int(width) * int(height)
        spp = self.spp if spp is None else int(spp)
        if pixels is None:
            if n is not None and int(n) != numpix:
                raise TptError("draw_samples: without pixels n must be width * height")
            n = numpix
        else:
            n = _entries("draw_samples", "pixels", pixels, n, ())
        if n < 0:
            raise TptError("draw_samples: n < 0")
        sum4, sq4, stream = self._sums_outputs("draw_samples", pixels, n, sum4, sq4, stream, pixels)
        (pp, ps, pq), on_dev, _keep = _buffer_ptrs(
            "draw_samples", [("pixels", pixels, "int32", 1), ("sum4", sum4, "float32", 4), ("sq4", sq4, "float32", 4)], n)
        total = self._call("tpt_draw_samples", want_rays, stream, int(frame), int(width), int(height), pp, n, spp, ps, pq,
                           1 if on_dev else 0)
        return ((sum4, sq4), total) if want_rays else (sum4, sq4)

    def _sums_outputs(self, what: str, like, n: int, sum4, sq4, stream: int, *inputs):
        """(sum4, sq4, stream) of a sums call (draw_samples, trace_samples) with the caller's `inputs` buffers: missing
        outputs allocated zeroed, of the kind of `like` (a CUDA tensor on the context's device for None or a DevicePtr),
        and the stream the call runs on."""
        if sum4 is None and sq4 is not None:
            raise TptError(f"{what}: sq4 needs sum4")
        alloc_dev = None
        if sum4 is None:
            if isinstance(like, np.ndarray):
                sum4, sq4 = np.zeros((n, 4), np.float32), np.zeros((n, 4), np.float32)
            else:
                import torch
                alloc_dev = like.device if hasattr(like, "device") else torch.device("cuda", self.device)
        # Torch CUDA tensors are written and read on torch's streams, which the library does not know: without an
        # explicit stream the call runs on torch's current stream of their device, after the torch work that filled
        # them (and the zeroing of outputs allocated here) and before the torch work that reads the sums.
        tdev = _cuda_device(*inputs, sum4, sq4) or (alloc_dev if alloc_dev is not None and alloc_dev.type == "cuda" else None)
        explicit = bool(stream)
        if tdev is not None and not explicit:
            stream = _torch_stream(tdev)
        if alloc_dev is not None:
            import contextlib
            import torch
            # outputs for an explicit stream are zeroed on it, so the call cannot overtake the fill
            other = explicit and alloc_dev.type == "cuda" and stream != _torch_stream(alloc_dev)
            on = torch.cuda.stream(torch.cuda.ExternalStream(stream, device=alloc_dev)) if other else contextlib.nullcontext()
            with on:
                sum4 = torch.zeros((n, 4), dtype=torch.float32, device=alloc_dev)
                sq4 = torch.zeros((n, 4), dtype=torch.float32, device=alloc_dev)
        return sum4, sq4, stream

    def trace_samples(self, inputs, ids=None, points: bool = False, entries=None, spp: int = 4, frame: int = 0, sum4=None,
                      sq4=None, stream: int = 0, want_rays: bool = True, n=None, num_in=None):
        """tpt_trace_samples: `spp` more samples of trace_rays (points False: `inputs` are rays {o.xyz, d.xyz}) or
        trace_irradiance (points True: surface points {p.xyz, n.xyz}, `ids` their sphere ids or None) for each entry of
        `entries` — int32 indices into inputs, duplicates and any order allowed; None = every input — ADDED to sum4
        (sum v.r, v.g, v.b, sample count) and, when given, sq4 (sum v.r^2, v.g^2, v.b^2, 0), both (N, 4) float32, v being
        the radiance (rays) or pi x the white-Lambert radiance (points). Sample s of input i at `frame` is the mean call's
        own (stream pixel_seed(i * spp + s, frame)), so an all-input call traces trace_rays' / trace_irradiance's samples
        at the same spp and frame. An input those calls do not trace adds no sample and no rays. Buffers are numpy
        arrays, torch tensors (CPU or CUDA) or DevicePtr (DevicePtr inputs need `num_in`, a DevicePtr list `n`), all host
        or all device. Allocation of missing sums (of the kind of `inputs`), streams and the return value are those of
        draw_samples. A call with a list is synchronous."""
        what = "trace_samples"
        if isinstance(inputs, DevicePtr) and num_in is None:
            raise TptError("trace_samples: DevicePtr inputs need num_in")
        num_in = _entries(what, "inputs", inputs, num_in, (6,))
        if ids is not None:
            if not points:
                raise TptError("trace_samples: ids are only taken with points")
            _entries(what, "ids", ids, num_in, ())
        if entries is None:
            if n is not None and int(n) != num_in:
                raise TptError("trace_samples: without entries n must be num_in")
            n = num_in
        else:
            n = _entries(what, "entries", entries, n, ())
        sum4, sq4, stream = self._sums_outputs(what, inputs, n, sum4, sq4, stream, inputs, ids, entries)
        (pi, pd), in_dev, _keep = _buffer_ptrs(what, [("inputs", inputs, "float32", 6), ("ids", ids, "int32", 1)], num_in)
        (pe, ps, pq), out_dev, _keep_out = _buffer_ptrs(
            what, [("entries", entries, "int32", 1), ("sum4", sum4, "float32", 4), ("sq4", sq4, "float32", 4)], n)
        if in_dev != out_dev:
            raise TptError("trace_samples: inputs, ids, entries, sum4 and sq4 must be all host or all device buffers")
        total = self._call("tpt_trace_samples", want_rays, stream, pi, pd, 1 if points else 0, num_in, pe, n, int(spp),
                           int(frame), ps, pq, 1 if in_dev else 0)
        return ((sum4, sq4), total) if want_rays else (sum4, sq4)

    @staticmethod
    def _adaptive_rounds(call, base_spp: int, max_spp: int, rel_err: float, frame: int, shape):
        """The round loop of render_adaptive and trace_adaptive: call(frame, entries or None) -> ((sum4, sq4), rays) adds
        base_spp samples per entry. One all-entry pass at `frame`, then rounds at frame + 1, ... over the entries
        adaptive_pixels picks (`shape`: its dilation grid), until it picks none or every entry has max_spp. Entries the
        first pass gave no sample (untraceable inputs) are shown to the rule as finished, with max_spp samples and no
        variance, so they are neither picked nor grow the picked set. Returns (sum4, rays)."""
        import torch
        (s, q), rays = call(frame, None)
        dead = (s[:, 3] == 0).unsqueeze(1)
        finished = torch.tensor([0.0, 0.0, 0.0, float(max_spp)], dtype=s.dtype, device=s.device)
        for f in range(frame + 1, frame + 1 + (max_spp - base_spp) // base_spp):
            idx = adaptive_pixels(torch.where(dead, finished, s), q, rel_err, max_spp, shape)
            if idx.numel() == 0:
                break
            (ds, dq), r = call(f, idx)
            s.index_add_(0, idx.long(), ds)
            q.index_add_(0, idx.long(), dq)
            rays += r
        return s, rays

    def trace_adaptive(self, inputs, ids=None, points: bool = False, base_spp: int = 4, max_spp: int = 64,
                       rel_err: float = 0.05, frame: int = 0, shape: Optional[Tuple[int, int]] = None):
        """Adaptive trace_rays (points False) or trace_irradiance (points True) on the device: one trace_samples pass over
        every input at base_spp (frame `frame`), then rounds at frames frame + 1, frame + 2, ... that give base_spp more
        samples to the inputs adaptive_pixels picks, until it picks none or every input has max_spp. shape = (h, w)
        declares that the N inputs form a row-major h x w grid (an equirect panorama, a lightmap's texels): the rule then
        grows the picked set by each picked entry's 3 x 3 neighbourhood, as render_adaptive does; without it there is no
        dilation. `inputs` and `ids` are (N, 6) float32 and (N,) int32 arrays or tensors (copied to the context's device
        if they are elsewhere). Untraceable inputs get no sample: they report 0 samples and a zero mean. Returns (mean
        float32 (N, 4) with alpha 0, samples per input int32 (N,), rays traced), all but the ray count CUDA tensors."""
        import torch
        if base_spp < 1 or max_spp < base_spp:
            raise TptError("trace_adaptive: need 1 <= base_spp <= max_spp")
        dev = torch.device("cuda", self.device)
        inputs = torch.as_tensor(inputs, device=dev)
        ids = None if ids is None else torch.as_tensor(ids, device=dev)
        n = _entries("trace_adaptive", "inputs", inputs, None, (6,))
        if shape is not None and int(shape[0]) * int(shape[1]) != n:
            raise TptError("trace_adaptive: shape does not hold N inputs")
        # every buffer is a CUDA tensor, so each trace_samples call runs on torch's current stream
        s, rays = self._adaptive_rounds(lambda f, idx: self.trace_samples(inputs, ids, points, idx, base_spp, f),
                                        base_spp, max_spp, rel_err, frame, shape)
        mean = torch.zeros((n, 4), dtype=torch.float32, device=dev)
        mean[:, :3] = s[:, :3] / s[:, 3:].clamp(min=1.0)
        return mean, s[:, 3].round().to(torch.int32), rays

    def render_adaptive(self, width: int, height: int, base_spp: int = 4, max_spp: int = 64, rel_err: float = 0.05,
                        frame: int = 0):
        """Adaptive fast-mode render on the device: one draw_samples pass over every pixel at base_spp (frame `frame`),
        then rounds at frames frame + 1, frame + 2, ... that give base_spp more samples to the pixels adaptive_pixels
        picks, until it picks none or every pixel has max_spp. Returns (image float32 [h, w, 4] with alpha 0, samples
        per pixel int32 [h, w], rays traced), all but the ray count CUDA tensors on the context's device. Every step —
        the library calls, the rule, the index conversion and the scatter of the sums — runs on torch's current stream."""
        import torch
        if base_spp < 1 or max_spp < base_spp:
            raise TptError("render_adaptive: need 1 <= base_spp <= max_spp")
        dev = torch.device("cuda", self.device)
        # every buffer is a CUDA tensor, so each draw_samples call runs on torch's current stream
        s, rays = self._adaptive_rounds(lambda f, idx: self.draw_samples(f, width, height, idx, base_spp),
                                        base_spp, max_spp, rel_err, frame, (height, width))
        image = torch.zeros((height, width, 4), dtype=torch.float32, device=dev)
        image.view(-1, 4)[:, :3] = s[:, :3] / s[:, 3:]
        return image, s[:, 3].round().to(torch.int32).view(height, width), rays

    def read_ray_count(self, stream: int = 0) -> int:
        out = ctypes.c_longlong(0)
        self._check(self._L.tpt_read_ray_count(self._h, ctypes.c_void_p(stream) if stream else None, ctypes.byref(out)),
                    "tpt_read_ray_count")
        return int(out.value)

    def last_kernel_ms(self) -> float:
        out = ctypes.c_float(0)
        self._check(self._L.tpt_last_kernel_ms(self._h, ctypes.byref(out)), "tpt_last_kernel_ms")
        return float(out.value)

    def last_launch_count(self) -> int:
        return int(self._L.tpt_last_launch_count(self._h))

    def last_scene_upload_bytes(self) -> int:
        """Bytes the most recent set_scene copied to the device (0: the scene was already resident)."""
        return int(self._L.tpt_last_scene_upload_bytes(self._h))

    # ---- device memory shared between ranks (CUDA IPC), see include/tpt_b200.h
    def mem_alloc(self, nbytes: int) -> DevicePtr:
        p = ctypes.c_void_p()
        self._check(self._L.tpt_mem_alloc(self._h, nbytes, ctypes.byref(p)), "tpt_mem_alloc")
        return DevicePtr(p.value)

    def mem_free(self, ptr: DevicePtr):
        self._check(self._L.tpt_mem_free(self._h, ctypes.c_void_p(ptr.addr)), "tpt_mem_free")

    def mem_to_host(self, ptr: DevicePtr, out: np.ndarray):
        self._check(self._L.tpt_mem_copy(self._h, out.ctypes.data, ctypes.c_void_p(ptr.addr), out.nbytes, 2), "tpt_mem_copy")
        return out

    def mem_from_host(self, ptr: DevicePtr, src: np.ndarray):
        src = np.ascontiguousarray(src)
        self._check(self._L.tpt_mem_copy(self._h, ctypes.c_void_p(ptr.addr), src.ctypes.data, src.nbytes, 1), "tpt_mem_copy")

    def ipc_export(self, ptr: DevicePtr) -> bytes:
        h = ctypes.create_string_buffer(64)
        self._check(self._L.tpt_ipc_export(self._h, ctypes.c_void_p(ptr.addr), h), "tpt_ipc_export")
        return bytes(h.raw)

    def ipc_open(self, handle: bytes) -> DevicePtr:
        p = ctypes.c_void_p()
        self._check(self._L.tpt_ipc_open(self._h, handle, ctypes.byref(p)), "tpt_ipc_open")
        return DevicePtr(p.value)

    def ipc_close(self, ptr: DevicePtr):
        self._check(self._L.tpt_ipc_close(self._h, ctypes.c_void_p(ptr.addr)), "tpt_ipc_close")

    def debug_libm(self, fn: int, x: np.ndarray) -> np.ndarray:
        """Device-side libm restatement of the exact mode: fn 0 sinf, 1 cosf, 2 powf(x,5)."""
        x = np.ascontiguousarray(x, np.float32)
        out = np.empty_like(x)
        self._check(self._L.tpt_debug_libm(self._h, fn, x.ctypes.data, out.ctypes.data, x.size), "tpt_debug_libm")
        return out

    def debug_hit(self, kform: int, rays: np.ndarray):
        """Nearest hit of rays[n, 6] = {o.xyz, d.xyz} with sweep form `kform` of the fast kernels -> (ids int32, t float32)."""
        rays = np.ascontiguousarray(rays, np.float32).reshape(-1, 6)
        ids = np.empty(len(rays), np.int32)
        t = np.empty(len(rays), np.float32)
        self._check(self._L.tpt_debug_hit(self._h, kform, rays.ctypes.data, ids.ctypes.data, t.ctypes.data, len(rays)), "tpt_debug_hit")
        return ids, t

    def last_kernels(self):
        """Trace kernels the calling thread's most recent draw / trace_rays / trace_irradiance / trace_samples /
        draw_samples / AOV call launched, as
        readable template instances (kernel_signature), in launch order. The library names the first 16 launches; past
        that the list ends with "... N more launches" (see tpt_debug_last_kernels)."""
        buf = ctypes.create_string_buffer(4096)
        n = self._L.tpt_debug_last_kernels(self._h, buf, len(buf))
        if n < 0:
            self._check(-n, "tpt_debug_last_kernels")
        names = [kernel_signature(s) for s in buf.value.decode().split("\n")] if n else []
        return names + ([f"... {n - len(names)} more launches"] if n > len(names) else [])

    def tonemap_srgb8(self, image, width: int, height: int) -> np.ndarray:
        addr, on_dev, _keep = _as_ptr(image)
        out = np.empty((height, width, 4), np.uint8)
        self._check(self._L.tpt_tonemap_srgb8(self._h, ctypes.c_void_p(addr), 1 if on_dev else 0, width, height,
                                              out.ctypes.data, 0, None), "tpt_tonemap_srgb8")
        return out

    def tonemap_rgba8(self, image, width: int, height: int, transfer: int = 0, bgr: bool = False, flip_y: bool = True) -> np.ndarray:
        """transfer 0: LinearToSRGB (PixelShader.hlsl), 1: sqrt gamma (Emscripten/main.cpp:67-79), 2: the C# TGA writer's
        (Cs/Program.cs:34-68; use bgr=True, flip_y=False for its byte layout)."""
        addr, on_dev, _keep = _as_ptr(image)
        out = np.empty((height, width, 4), np.uint8)
        self._check(self._L.tpt_tonemap_rgba8(self._h, ctypes.c_void_p(addr), 1 if on_dev else 0, width, height,
                                              out.ctypes.data, 0, transfer, 1 if bgr else 0, 1 if flip_y else 0, None),
                    "tpt_tonemap_rgba8")
        return out


# ---- the reference's Test.h API (C++-mangled symbols of the drop-in shim) -----------------------------------
def _load_shim():
    global _shim
    if _shim is not None:
        return _shim
    _load_lib()
    if not os.path.exists(SHIM_PATH):
        raise TptError(f"{SHIM_PATH} is missing: build with `make -C toypathtracer_b200/csrc`")
    S = ctypes.CDLL(SHIM_PATH)
    ci, cu, cf, vp = ctypes.c_int, ctypes.c_uint, ctypes.c_float, ctypes.c_void_p
    S._Z14InitializeTestv.argtypes = []; S._Z14InitializeTestv.restype = None
    S._Z12ShutdownTestv.argtypes = []; S._Z12ShutdownTestv.restype = None
    S._Z10UpdateTestfiiij.argtypes = [cf, ci, ci, ci, cu]; S._Z10UpdateTestfiiij.restype = None
    S._Z8DrawTestfiiiPfRij.argtypes = [cf, ci, ci, ci, vp, ctypes.POINTER(ci), cu]; S._Z8DrawTestfiiiPfRij.restype = None
    S._Z14GetObjectCountRiS_S_S_.argtypes = [ctypes.POINTER(ci)] * 4; S._Z14GetObjectCountRiS_S_S_.restype = None
    S._Z12GetSceneDescPvS_S_S_Pi.argtypes = [vp, vp, vp, vp, ctypes.POINTER(ci)]; S._Z12GetSceneDescPvS_S_S_Pi.restype = None
    S.tpt_shim_set_mode.argtypes = [ci]; S.tpt_shim_set_mode.restype = None
    S.tpt_shim_reset_scene.argtypes = []; S.tpt_shim_reset_scene.restype = None
    S.tpt_shim_set_variant.argtypes = [ci, ci]; S.tpt_shim_set_variant.restype = None
    _shim = S
    return S


def InitializeTest():
    """Test.h:10 — creates the CUDA context (the reference creates its CPU task scheduler here)."""
    _load_shim()._Z14InitializeTestv()


def ShutdownTest():
    """Test.h:11"""
    _load_shim()._Z12ShutdownTestv()


def UpdateTest(time: float, frameCount: int, screenWidth: int, screenHeight: int, testFlags: int = 0):
    """Test.h:13 — host-side scene animation, camera, emissive list; uploads the scene to the device."""
    _load_shim()._Z10UpdateTestfiiij(time, frameCount, screenWidth, screenHeight, testFlags)


def DrawTest(time: float, frameCount: int, screenWidth: int, screenHeight: int, backbuffer: np.ndarray,
             testFlags: int = 0) -> int:
    """Test.h:14 — renders one frame into the caller-owned float RGBA backbuffer; returns outRayCount."""
    if not (isinstance(backbuffer, np.ndarray) and backbuffer.dtype == np.float32 and backbuffer.flags["C_CONTIGUOUS"]
            and backbuffer.size == screenWidth * screenHeight * 4):
        raise TptError("backbuffer must be a C-contiguous float32 array of width*height*4")
    rc = ctypes.c_int(0)
    _load_shim()._Z8DrawTestfiiiPfRij(time, frameCount, screenWidth, screenHeight, backbuffer.ctypes.data,
                                      ctypes.byref(rc), testFlags)
    return int(rc.value)


def GetObjectCount() -> Tuple[int, int, int, int]:
    """Test.h:16 -> (count, objectSize, materialSize, camSize)"""
    v = [ctypes.c_int(0) for _ in range(4)]
    _load_shim()._Z14GetObjectCountRiS_S_S_(*[ctypes.byref(x) for x in v])
    return tuple(int(x.value) for x in v)


def GetSceneDesc():
    """Test.h:17 -> (spheres[n] SPHERE_DTYPE, materials[n] MATERIAL_DTYPE, camera CAMERA_DTYPE, emissive ids)."""
    n, so, sm, sc = GetObjectCount()
    spheres = np.zeros(n, SPHERE_DTYPE); mats = np.zeros(n, MATERIAL_DTYPE); cam = np.zeros(1, CAMERA_DTYPE)
    em = np.zeros(max(n, 1), np.int32); ec = ctypes.c_int(0)
    _load_shim()._Z12GetSceneDescPvS_S_S_Pi(spheres.ctypes.data, mats.ctypes.data, cam.ctypes.data, em.ctypes.data,
                                            ctypes.byref(ec))
    return spheres, mats, cam, em[: ec.value].copy()


def reset_scene():
    """Un-animated scene again (UpdateTest with kFlagAnimate moves spheres 1 and 8 permanently, Test.cpp:304-308)."""
    _load_shim().tpt_shim_reset_scene()


def set_variant(big_scene: bool = True, mitsuba_compare: bool = False):
    """The reference's compile-time switches DO_BIG_SCENE (Test.cpp:10-11: 46 vs 9 spheres) and DO_MITSUBA_COMPARE
    (Config.h:25: constant sky, zero Metal roughness, zero aperture) at run time; resets the scene."""
    _load_shim().tpt_shim_set_variant(1 if big_scene else 0, 1 if mitsuba_compare else 0)


def set_light_sampling(on: bool = True):
    """The reference's compile-time switch DO_LIGHT_SAMPLING (Config.h:24) at run time for the Test.h API: False renders
    without explicit light sampling (no shadow rays; every hit adds its emission). Takes effect with the next
    UpdateTest()."""
    _load_shim().tpt_shim_set_light_sampling(1 if on else 0)


def set_mode(mode: int):
    """Mode used by DrawTest(): MODE_EXACT (default, bit-identical to the reference) or MODE_FAST."""
    _load_shim().tpt_shim_set_mode(mode)


from .scenes import reference_scene, stress_scene, make_camera, camera_rays  # noqa: E402,F401
