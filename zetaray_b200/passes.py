"""Host-side mirrors of the reference's pass objects over the C-ABI (thin; no compute here).

Names follow ZetaRenderPass: GBufferRT, PreLighting, DirectLighting, IndirectLighting, Compositing,
TAA, AutoExposure, Display -- each with the reference's verbs (Init in the constructor, OnWindowResized, Render, GetOutput)."""
import ctypes as C
import numpy as np

from . import _lib
from ._lib import lib, check


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


class Scene:
    """Flat scene buffers + BVH on the device (zr_scene)."""

    def __init__(self, flat):
        self.flat = flat
        d = _lib.SceneDesc()
        self._keep = [np.ascontiguousarray(x) for x in (flat.vertices, flat.indices, flat.instances,
                                                        flat.instance_num_tris, flat.materials, flat.emissives)]
        v, i, inst, nt, m, e = self._keep
        d.h_vertices, d.num_vertices = _vp(v), len(v)
        d.h_indices, d.num_indices = _vp(i), len(i)
        d.h_instances, d.num_instances = _vp(inst), len(inst)
        d.h_instance_num_tris = _vp(nt)
        d.h_materials, d.num_materials = _vp(m), len(m)
        d.h_emissives, d.num_emissives = (_vp(e) if len(e) else None), len(e)
        self.handle = C.c_void_p()
        check(lib.zr_scene_create(C.byref(d), C.byref(self.handle)))

    def bvh_stats(self):
        out = (C.c_uint32 * 4)()
        check(lib.zr_scene_bvh_stats(self.handle, out))
        return dict(nodes=out[0], tris=out[1], max_depth=out[2], bytes=out[3])

    def prelighting(self, stream=None):
        check(lib.zr_prelighting_render(self.handle, stream))

    def set_presampling(self, num_sets, set_size):
        """128 x 512 is what the reference enables at >= 13107 emissive triangles; 0, 0 = alias-table sampling."""
        check(lib.zr_scene_set_presampling(self.handle, num_sets, set_size))

    def presample(self, frame_num, stream=None):
        """PresampleEmissives: once per frame, before DirectLighting / IndirectLighting."""
        check(lib.zr_presample_emissives(self.handle, C.c_uint32(frame_num), stream))

    def sample_sets(self):
        p, n, m = C.c_void_p(), C.c_uint32(), C.c_uint32()
        check(lib.zr_scene_get_sample_sets(self.handle, C.byref(p), C.byref(n), C.byref(m)))
        out = np.zeros(n.value * m.value * 10, dtype=np.uint32)
        if out.size:
            check(lib.zr_memcpy_d2h(_vp(out), p, C.c_size_t(out.nbytes), None))
            check(lib.zr_stream_synchronize(None))
        return out

    def set_light_voxel_grid(self, grid_dim, extents, offset_y=0.0):
        """Reference defaults: (32, 8, 40) voxels of half-extents (0.6, 0.45, 0.6); (0, 0, 0) switches the grid off."""
        d = (C.c_uint32 * 3)(*grid_dim)
        e = (C.c_float * 3)(*extents)
        check(lib.zr_scene_set_light_voxel_grid(self.handle, d, e, C.c_float(offset_y)))

    def build_light_voxel_grid(self, fc, stream=None):
        """BuildLightVoxelGrid: once per frame (the grid follows the camera), after presample()."""
        check(lib.zr_build_light_voxel_grid(self.handle, C.byref(fc), stream))

    def light_voxel_grid(self):
        p, n = C.c_void_p(), C.c_uint32()
        check(lib.zr_scene_get_light_voxel_grid(self.handle, C.byref(p), C.byref(n)))
        out = np.zeros(n.value * 8, dtype=np.uint32)
        if out.size:
            check(lib.zr_memcpy_d2h(_vp(out), p, C.c_size_t(out.nbytes), None))
            check(lib.zr_stream_synchronize(None))
        return out

    def alias_table(self):
        p = C.c_void_p()
        n = C.c_uint32()
        check(lib.zr_scene_get_alias_table(self.handle, C.byref(p), C.byref(n)))
        out = np.zeros(n.value, dtype=np.dtype([("CachedP_Orig", "<f4"), ("CachedP_Alias", "<f4"), ("P_Curr", "<f4"), ("Alias", "<u4")]))
        if n.value:
            check(lib.zr_memcpy_d2h(_vp(out), p, C.c_size_t(out.nbytes), None))
            check(lib.zr_stream_synchronize(None))
        return out

    def close(self):
        if self.handle:
            lib.zr_scene_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class GBuffers:
    """The renderer-owned, double-buffered G-buffer planes (DefaultRendererImpl.h:111-121)."""

    def __init__(self, w, h, with_tridiff=False):
        self.w, self.h = w, h
        self.g = [_lib.GBuffer(), _lib.GBuffer()]
        for g in self.g:
            check(lib.zr_gbuffer_alloc(w, h, int(with_tridiff), C.byref(g)))
        self.curr = 0

    def flip(self):
        self.curr ^= 1

    def fill_inputs(self, fi):
        fi.curr = self.g[self.curr]
        fi.prev = self.g[self.curr ^ 1]

    def download(self, which="curr"):
        g = self.g[self.curr if which == "curr" else self.curr ^ 1]
        n = self.w * self.h
        core = np.zeros((n, 4), dtype=np.uint32)
        depth = np.zeros(n, dtype=np.float32)
        me = np.zeros((n, 2), dtype=np.uint32)
        coat = np.zeros((n, 2), dtype=np.uint32)
        for arr, p in ((core, g.d_core), (depth, g.d_depth), (me, g.d_motion_emissive), (coat, g.d_coat)):
            check(lib.zr_memcpy_d2h(_vp(arr), C.c_void_p(p), C.c_size_t(arr.nbytes), None))
        td = None
        if g.d_tridiff:
            td = np.zeros((n, 6), dtype=np.uint32)
            check(lib.zr_memcpy_d2h(_vp(td), C.c_void_p(g.d_tridiff), C.c_size_t(td.nbytes), None))
        check(lib.zr_stream_synchronize(None))
        return core, depth, me, coat, td

    def close(self):
        for g in self.g:
            lib.zr_gbuffer_free(C.byref(g))


def download_image(img, dtype, comps):
    out = np.zeros((img.width * img.height, comps), dtype=dtype)
    assert out.nbytes == img.height * img.pitch_bytes, (out.nbytes, img.height, img.pitch_bytes)
    check(lib.zr_memcpy_d2h(_vp(out), C.c_void_p(img.d_ptr), C.c_size_t(out.nbytes), None))
    check(lib.zr_stream_synchronize(None))
    return out


def download_image_pitched(img, dtype, comps):
    """An image whose rows are padded (pitch_bytes > width * texel_bytes): downloads the pitched rows and crops them."""
    item = np.dtype(dtype).itemsize * comps
    assert img.texel_bytes == item and img.pitch_bytes % item == 0
    raw = np.zeros((img.height, img.pitch_bytes // item, comps), dtype=dtype)
    check(lib.zr_memcpy_d2h(_vp(raw), C.c_void_p(img.d_ptr), C.c_size_t(raw.nbytes), None))
    check(lib.zr_stream_synchronize(None))
    return np.ascontiguousarray(raw[:, :img.width]).reshape(img.width * img.height, comps)


class _Pass:
    prefix = None

    def __del__(self):
        try:
            if getattr(self, "handle", None):
                getattr(lib, self.prefix + "_destroy")(self.handle)
                self.handle = None
        except Exception:
            pass


class GBufferRT(_Pass):
    prefix = "zr_gbuffer_pass"

    def __init__(self):
        self.handle = C.c_void_p()
        check(lib.zr_gbuffer_pass_create(C.byref(self.handle)))

    def SetRows(self, y0, y1):
        check(lib.zr_gbuffer_pass_set_rows(self.handle, y0, y1))

    def Render(self, fi, stream=None):
        check(lib.zr_gbuffer_pass_render(self.handle, C.byref(fi), stream))


class DirectLighting(_Pass):
    prefix = "zr_direct_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_direct_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.DirectParams()
        check(lib.zr_direct_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        check(lib.zr_direct_pass_set_params(self.handle, C.byref(self.params)))

    def OnWindowResized(self, w, h):
        check(lib.zr_direct_pass_resize(self.handle, w, h))

    def ResetTemporal(self):
        check(lib.zr_direct_pass_reset_temporal(self.handle))

    def SetRows(self, y0, y1):
        check(lib.zr_direct_pass_set_rows(self.handle, y0, y1))

    def SetHaloExchange(self, fn):
        """fn: a _lib.HALO_EXCHANGE_FN instance (kept alive here) or None."""
        self._halo_fn = fn
        check(lib.zr_direct_pass_set_halo_exchange(self.handle, fn if fn is not None else _lib.HALO_EXCHANGE_FN(), None))

    def SetCostMap(self, d_cycles):
        check(lib.zr_direct_pass_set_cost_map(self.handle, C.c_void_p(d_cycles)))

    def SetScheduleCosts(self, tile_costs, tiles_x, tiles_y):
        """tile_costs: sequence of tiles_x * tiles_y floats (row-major) or None."""
        arr = None if tile_costs is None else (C.c_double * (tiles_x * tiles_y))(*tile_costs)
        check(lib.zr_direct_pass_set_schedule_costs(self.handle, arr, tiles_x, tiles_y))

    def Render(self, fi, stream=None):
        check(lib.zr_direct_pass_render(self.handle, C.byref(fi), stream))

    def GetOutput(self, which=0):
        img = _lib.Image2D()
        check(lib.zr_direct_pass_get_output(self.handle, which, C.byref(img)))
        return img


class IndirectLighting(_Pass):
    prefix = "zr_indirect_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_indirect_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.IndirectParams()
        check(lib.zr_indirect_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        check(lib.zr_indirect_pass_set_params(self.handle, C.byref(self.params)))

    def OnWindowResized(self, w, h):
        check(lib.zr_indirect_pass_resize(self.handle, w, h))

    def ResetTemporal(self):
        check(lib.zr_indirect_pass_reset_temporal(self.handle))

    def SetRows(self, y0, y1):
        check(lib.zr_indirect_pass_set_rows(self.handle, y0, y1))

    def SetHaloExchange(self, fn):
        self._halo_fn = fn
        check(lib.zr_indirect_pass_set_halo_exchange(self.handle, fn if fn is not None else _lib.HALO_EXCHANGE_FN(), None))

    def SetCostMap(self, d_cycles):
        check(lib.zr_indirect_pass_set_cost_map(self.handle, C.c_void_p(d_cycles)))

    def SetScheduleCosts(self, tile_costs, tiles_x, tiles_y):
        arr = None if tile_costs is None else (C.c_double * (tiles_x * tiles_y))(*tile_costs)
        check(lib.zr_indirect_pass_set_schedule_costs(self.handle, arr, tiles_x, tiles_y))

    def Render(self, fi, stream=None):
        check(lib.zr_indirect_pass_render(self.handle, C.byref(fi), stream))

    def GetOutput(self, which=0):
        img = _lib.Image2D()
        check(lib.zr_indirect_pass_get_output(self.handle, which, C.byref(img)))
        return img


class IndirectLightingGI(_Pass):
    """IndirectLighting with INTEGRATOR::ReSTIR_GI (zr_gi_pass, csrc/rgi.cu)."""
    prefix = "zr_gi_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_gi_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.GIParams()
        check(lib.zr_gi_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        check(lib.zr_gi_pass_set_params(self.handle, C.byref(self.params)))

    PATH_TRACING, RESTIR_GI = 0, 1

    def SetMethod(self, integrator):
        """IndirectLighting::SetMethod for the two integrators this pass object runs: the plain path tracer
        (PathTracer.hlsl) or ReSTIR GI."""
        check(lib.zr_gi_pass_set_method(self.handle, int(integrator)))

    def SetRows(self, y0, y1):
        check(lib.zr_gi_pass_set_rows(self.handle, y0, y1))

    def SetHaloExchange(self, fn):
        self._hook = fn
        check(lib.zr_gi_pass_set_halo_exchange(self.handle, fn if fn is not None else _lib.HALO_EXCHANGE_FN(), None))

    def OnWindowResized(self, w, h):
        check(lib.zr_gi_pass_resize(self.handle, w, h))

    def ResetTemporal(self):
        check(lib.zr_gi_pass_reset_temporal(self.handle))

    def Render(self, fi, stream=None):
        check(lib.zr_gi_pass_render(self.handle, C.byref(fi), stream))

    def GetOutput(self, which=0):
        img = _lib.Image2D()
        check(lib.zr_gi_pass_get_output(self.handle, which, C.byref(img)))
        return img


class Compositing(_Pass):
    prefix = "zr_compositing_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_compositing_pass_create(w, h, C.byref(self.handle)))

    def SetParams(self, emissive_di=1, indirect=1, firefly_filter=1):
        p = _lib.CompositingParams(emissive_di, indirect, firefly_filter)
        check(lib.zr_compositing_pass_set_params(self.handle, C.byref(p)))

    def SetRows(self, y0, y1):
        check(lib.zr_compositing_pass_set_rows(self.handle, y0, y1))

    def Render(self, fi, d_direct, d_indirect, stream=None):
        check(lib.zr_compositing_pass_render(self.handle, C.byref(fi), C.c_void_p(d_direct), C.c_void_p(d_indirect), stream))

    def GetOutput(self):
        img = _lib.Image2D()
        check(lib.zr_compositing_pass_get_output(self.handle, C.byref(img)))
        return img


class TAA(_Pass):
    prefix = "zr_taa_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_taa_pass_create(w, h, C.byref(self.handle)))

    def SetRows(self, y0, y1):
        check(lib.zr_taa_pass_set_rows(self.handle, y0, y1))

    def Render(self, fi, d_signal, stream=None):
        check(lib.zr_taa_pass_render(self.handle, C.byref(fi), C.c_void_p(d_signal), stream))

    def GetOutput(self):
        img = _lib.Image2D()
        check(lib.zr_taa_pass_get_output(self.handle, C.byref(img)))
        return img


class SVGF(_Pass):
    """SVGF denoiser (zr_svgf_pass_*): RGBA32F signal in, RGBA32F out (alpha = filtered variance); between Compositing and TAA."""
    prefix = "zr_svgf_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_svgf_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.SvgfParams()
        check(lib.zr_svgf_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        for k, v in kw.items():
            setattr(self.params, k, v)
        check(lib.zr_svgf_pass_set_params(self.handle, C.byref(self.params)))

    def ResetTemporal(self):
        check(lib.zr_svgf_pass_reset_temporal(self.handle))

    def Render(self, fi, d_signal, stream=None):
        check(lib.zr_svgf_pass_render(self.handle, C.byref(fi), C.c_void_p(d_signal), stream))

    def GetOutput(self, which=0):
        img = _lib.Image2D()
        check(lib.zr_svgf_pass_get_output(self.handle, which, C.byref(img)))
        return img


class AutoExposure(_Pass):
    """AutoExposure (zr_auto_exposure_pass, csrc/display.cu): luminance histogram of the TAA input -> adapted exposure.
    GetOutput() is the 1 x 1 float2 {exposure, adapted luminance}; Render reads the frame's dt (seconds)."""
    prefix = "zr_auto_exposure_pass"

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_auto_exposure_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.AutoExposureParams()
        check(lib.zr_auto_exposure_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        p = _lib.AutoExposureParams.from_buffer_copy(self.params)
        for k, v in kw.items():
            setattr(p, k, v)
        check(lib.zr_auto_exposure_pass_set_params(self.handle, C.byref(p)))
        self.params = p

    def OnWindowResized(self, w, h):
        check(lib.zr_auto_exposure_pass_resize(self.handle, w, h))

    def ResetTemporal(self):
        check(lib.zr_auto_exposure_pass_reset_temporal(self.handle))

    def SetRows(self, y0, y1):
        check(lib.zr_auto_exposure_pass_set_rows(self.handle, y0, y1))

    def SetReduce(self, fn):
        """fn: a _lib.REDUCE_U32_FN instance (kept alive here) or None."""
        self._reduce_fn = fn
        check(lib.zr_auto_exposure_pass_set_reduce(self.handle, fn if fn is not None else _lib.REDUCE_U32_FN(), None))

    def Render(self, fi, d_signal, stream=None):
        check(lib.zr_auto_exposure_pass_render(self.handle, C.byref(fi), C.c_void_p(d_signal), stream))

    def GetOutput(self):
        img = _lib.Image2D()
        check(lib.zr_auto_exposure_pass_get_output(self.handle, C.byref(img)))
        return img


class Display(_Pass):
    """Display (zr_display_pass, csrc/display.cu): TAA output x exposure -> tone mapper -> sRGB RGBA8."""
    prefix = "zr_display_pass"
    NONE, NEUTRAL, AGX_DEFAULT, AGX_GOLDEN, AGX_PUNCHY, AGX_CUSTOM = range(6)

    def __init__(self, w, h):
        self.handle = C.c_void_p()
        check(lib.zr_display_pass_create(w, h, C.byref(self.handle)))
        self.params = _lib.DisplayParams()
        check(lib.zr_display_pass_default_params(C.byref(self.params)))

    def SetParams(self, **kw):
        p = _lib.DisplayParams.from_buffer_copy(self.params)
        for k, v in kw.items():
            setattr(p, k, v)
        check(lib.zr_display_pass_set_params(self.handle, C.byref(p)))
        self.params = p

    def SetLUT(self, lut):
        """lut: the Tony McMapface LUT as packed R9G9B9E5 texels, uint32[48][48][48] (x fastest)."""
        a = np.ascontiguousarray(lut, dtype=np.uint32)
        check(lib.zr_display_pass_set_lut(self.handle, _vp(a), C.c_uint32(a.shape[0] if a.ndim == 3 else 0)))

    def OnWindowResized(self, w, h):
        check(lib.zr_display_pass_resize(self.handle, w, h))

    def SetRows(self, y0, y1):
        check(lib.zr_display_pass_set_rows(self.handle, y0, y1))

    def Render(self, fi, d_signal, d_exposure, stream=None):
        check(lib.zr_display_pass_render(self.handle, C.byref(fi), C.c_void_p(d_signal), C.c_void_p(d_exposure), stream))

    def GetOutput(self):
        img = _lib.Image2D()
        check(lib.zr_display_pass_get_output(self.handle, C.byref(img)))
        return img


class _Borrowed:
    """A pass handle owned by a Renderer: same verbs as the owning classes, never destroyed from here."""

    def __init__(self, cls, handle):
        self.__class__ = type("Borrowed" + cls.__name__, (cls,), {"__del__": lambda self: None})
        self.handle = handle
        if cls is DirectLighting:
            self.params = _lib.DirectParams()
            check(lib.zr_direct_pass_default_params(C.byref(self.params)))
        if cls is IndirectLighting:
            self.params = _lib.IndirectParams()
            check(lib.zr_indirect_pass_default_params(C.byref(self.params)))
        if cls is SVGF:
            self.params = _lib.SvgfParams()
            check(lib.zr_svgf_pass_default_params(C.byref(self.params)))
        if cls is AutoExposure:
            self.params = _lib.AutoExposureParams()
            check(lib.zr_auto_exposure_pass_default_params(C.byref(self.params)))
        if cls is Display:
            self.params = _lib.DisplayParams()
            check(lib.zr_display_pass_default_params(C.byref(self.params)))


class Comm:
    """zr_comm: halo transport between strips (NCCL, bound inside the library). `Comm.from_torch()` distributes the id through an
    initialised torch.distributed process group; any other out-of-band channel works with Comm.unique_id() / Comm(id, rank, world)."""

    def __init__(self, id256, rank, world):
        self.handle = C.c_void_p()
        self.rank, self.world = rank, world
        buf = (C.c_ubyte * 256).from_buffer_copy(bytes(id256))
        check(lib.zr_comm_create(buf, int(rank), int(world), C.byref(self.handle)))

    @staticmethod
    def unique_id():
        buf = (C.c_ubyte * 256)()
        check(lib.zr_comm_unique_id(buf))
        return bytes(buf)

    @classmethod
    def from_torch(cls, group=None):
        import torch
        import torch.distributed as dist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        dev = "cuda" if dist.get_backend(group) == "nccl" else "cpu"
        t = torch.zeros(256, dtype=torch.uint8)
        if rank == 0:
            t = torch.frombuffer(bytearray(cls.unique_id()), dtype=torch.uint8).clone()
        t = t.to(dev)
        dist.broadcast(t, 0, group=group)
        return cls(bytes(t.cpu().numpy().tobytes()), rank, world)

    def allreduce_u32(self, d_values, n, stream=None, which_comm=0):
        """In-place sum of n uint32 values (device pointer) over every rank."""
        check(lib.zr_comm_allreduce_u32(self.handle, int(which_comm), C.c_void_p(d_values), C.c_uint32(n), stream))

    def stats(self):
        b, c = C.c_uint64(), C.c_uint64()
        check(lib.zr_comm_stats(self.handle, C.byref(b), C.byref(c)))
        return b.value, c.value

    def close(self):
        if self.handle:
            lib.zr_comm_destroy(self.handle)
            self.handle = None


class Renderer:
    """The frame driver (zr_renderer, csrc/renderer.cu): G-buffers + all passes, one Render(frame constants) per frame."""

    def __init__(self, scene, w, h, two_streams=True, with_tridiff=False):
        self.scene = scene
        self.handle = C.c_void_p()
        desc = _lib.RendererDesc(w, h, int(with_tridiff), int(two_streams))
        check(lib.zr_renderer_create(C.byref(desc), scene.handle, C.byref(self.handle)))
        hs = [C.c_void_p() for _ in range(5)]
        check(lib.zr_renderer_get_passes(self.handle, *[C.byref(x) for x in hs]))
        self.gbuffer, self.direct, self.indirect, self.compositing, self.taa = (
            _Borrowed(cls, hnd) for cls, hnd in zip((GBufferRT, DirectLighting, IndirectLighting, Compositing, TAA), hs))

    def Render(self, fc, stream=None):
        check(lib.zr_renderer_render(self.handle, C.byref(fc), stream))

    PATH_TRACING, RESTIR_GI, RESTIR_PT = 0, 1, 2

    def SetMethod(self, integrator):
        """IndirectLighting::SetMethod as the renderer calls it (DefaultRenderer.cpp:243)."""
        check(lib.zr_renderer_set_integrator(self.handle, int(integrator)))
        if integrator != self.RESTIR_PT:
            h = C.c_void_p()
            check(lib.zr_renderer_get_gi_pass(self.handle, C.byref(h)))
            self.gi = _Borrowed(IndirectLightingGI, h)

    def SetShard(self, comm, bounds, gather_output=True):
        """Strip-sharded frame: this rank renders rows [bounds[rank], bounds[rank + 1]); None returns to the whole frame."""
        if comm is None:
            check(lib.zr_renderer_set_shard(self.handle, None, None, 0))
            return
        arr = (C.c_uint32 * len(bounds))(*[int(b) for b in bounds])
        check(lib.zr_renderer_set_shard(self.handle, comm.handle, arr, int(gather_output)))
        self._comm = comm

    def SetDenoiser(self, enable=True):
        """SVGF between Compositing and TAA (BASELINE config 3)."""
        h = C.c_void_p()
        check(lib.zr_renderer_set_denoiser(self.handle, int(enable), C.byref(h)))
        self.svgf = _Borrowed(SVGF, h) if enable else None

    def SetDisplay(self, enable=True, lut=None):
        """AutoExposure on the TAA input and Display on the TAA output (PostProcessor.cpp). lut: the Tony McMapface LUT the
        default NEUTRAL tone mapper needs (Display.SetLUT)."""
        ae, disp = C.c_void_p(), C.c_void_p()
        check(lib.zr_renderer_set_display(self.handle, int(enable), C.byref(ae), C.byref(disp)))
        self.auto_exposure = _Borrowed(AutoExposure, ae) if enable else None
        self.display = _Borrowed(Display, disp) if enable else None
        if enable and lut is not None:
            self.display.SetLUT(lut)

    def GetDisplayOutput(self):
        img = _lib.Image2D()
        check(lib.zr_renderer_get_display_output(self.handle, C.byref(img)))
        return img

    def ApplySceneSettings(self, use_lvg=False):
        """The reference's host decision: presampled sets iff >= 13107 emissive triangles, LVG only with them."""
        out = (C.c_uint32 * 2)()
        check(lib.zr_renderer_apply_scene_settings(self.handle, int(use_lvg), out))
        return bool(out[0]), bool(out[1])

    def GetOutput(self):
        img = _lib.Image2D()
        check(lib.zr_renderer_get_output(self.handle, C.byref(img)))
        return img

    def close(self):
        if self.handle:
            lib.zr_renderer_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
