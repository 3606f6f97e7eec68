"""Host-side mirrors of the reference's pass objects over the C-ABI (thin; no compute here).

Names follow ZetaRenderPass: GBufferRT, PreLighting, DirectLighting, IndirectLighting, Compositing,
TAA, AutoExposure, Display -- each with the reference's verbs (Init in the constructor, OnWindowResized, Render, GetOutput)."""
import ctypes as C
import numpy as np

from . import _lib
from ._lib import lib, check
from .scene import EMISSIVE_TRI, MATERIAL


def _vp(a):
    return a.ctypes.data_as(C.c_void_p)


def _d2h(*copies):
    """Copies every (host array, device pointer) pair into its array, waits for the copies and returns the arrays.
    An array that is None or empty is not copied."""
    for out, d_ptr in copies:
        if out is not None and out.nbytes:
            check(lib.zr_memcpy_d2h(_vp(out), d_ptr, out.nbytes, None))
    check(lib.zr_stream_synchronize(None))
    return tuple(out for out, _ in copies)


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

    def material_features(self):
        """ZR_MATERIAL_* bits of the current material table."""
        out = C.c_uint32()
        check(lib.zr_scene_material_features(self.handle, C.byref(out)))
        return out.value

    def update_materials(self, first, materials, stream=None):
        """Replaces materials [first, first + len(materials)) between frames (zr_scene_update_materials): the emissive triangles
        of changed lights take the new factor / strength on the device and the alias table is rebuilt on `stream`. Geometry,
        instances and the emissive set stay; scene.update_materials applies the same edit to a FlatScene."""
        m = np.ascontiguousarray(np.asarray(materials, dtype=MATERIAL).reshape(-1))
        check(lib.zr_scene_update_materials(self.handle, int(first), len(m), _vp(m), stream))

    def tables(self):
        """(materials, emissive triangles) as the device holds them."""
        dm, nm, de, ne = C.c_void_p(), C.c_uint32(), C.c_void_p(), C.c_uint32()
        check(lib.zr_scene_get_tables(self.handle, C.byref(dm), C.byref(nm), C.byref(de), C.byref(ne)))
        return _d2h((np.zeros(nm.value, dtype=MATERIAL), dm), (np.zeros(ne.value, dtype=EMISSIVE_TRI), de))

    def prelighting(self, stream=None):
        check(lib.zr_prelighting_render(self.handle, stream))

    def set_presampling(self, num_sets, set_size):
        """128 x 512 is what the reference enables at >= 13107 emissive triangles; 0, 0 = alias-table sampling."""
        check(lib.zr_scene_set_presampling(self.handle, num_sets, set_size))

    def presample(self, frame_num, stream=None):
        """PresampleEmissives: once per frame, before DirectLighting / IndirectLighting."""
        check(lib.zr_presample_emissives(self.handle, frame_num, stream))

    def sample_sets(self):
        p, n, m = C.c_void_p(), C.c_uint32(), C.c_uint32()
        check(lib.zr_scene_get_sample_sets(self.handle, C.byref(p), C.byref(n), C.byref(m)))
        return _d2h((np.zeros(n.value * m.value * 10, dtype=np.uint32), p))[0]

    def set_light_voxel_grid(self, grid_dim, extents, offset_y=0.0):
        """Reference defaults: (32, 8, 40) voxels of half-extents (0.6, 0.45, 0.6); (0, 0, 0) switches the grid off."""
        check(lib.zr_scene_set_light_voxel_grid(self.handle, (C.c_uint32 * 3)(*grid_dim), (C.c_float * 3)(*extents), offset_y))

    def build_light_voxel_grid(self, fc, stream=None):
        """BuildLightVoxelGrid: once per frame (the grid follows the camera), after presample()."""
        check(lib.zr_build_light_voxel_grid(self.handle, C.byref(fc), stream))

    def light_voxel_grid(self):
        p, n = C.c_void_p(), C.c_uint32()
        check(lib.zr_scene_get_light_voxel_grid(self.handle, C.byref(p), C.byref(n)))
        return _d2h((np.zeros(n.value * 8, dtype=np.uint32), p))[0]

    def alias_table(self):
        p, n = C.c_void_p(), C.c_uint32()
        check(lib.zr_scene_get_alias_table(self.handle, C.byref(p), C.byref(n)))
        return _d2h((np.zeros(n.value, dtype=_lib.ALIAS_ENTRY), p))[0]

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
        """(core, depth, motion_emissive, coat, tridiff or None) of the current or the previous G-buffer."""
        g = self.g[self.curr if which == "curr" else self.curr ^ 1]
        n = self.w * self.h
        return _d2h((np.zeros((n, 4), dtype=np.uint32), g.d_core), (np.zeros(n, dtype=np.float32), g.d_depth),
                    (np.zeros((n, 2), dtype=np.uint32), g.d_motion_emissive), (np.zeros((n, 2), dtype=np.uint32), g.d_coat),
                    (np.zeros((n, 6), dtype=np.uint32) if g.d_tridiff else None, g.d_tridiff))

    def close(self):
        for g in self.g:
            lib.zr_gbuffer_free(C.byref(g))


def download_image(img, dtype, comps):
    out = np.zeros((img.width * img.height, comps), dtype=dtype)
    assert out.nbytes == img.height * img.pitch_bytes, (out.nbytes, img.height, img.pitch_bytes)
    return _d2h((out, img.d_ptr))[0]


def download_image_pitched(img, dtype, comps):
    """An image whose rows are padded (pitch_bytes > width * texel_bytes): downloads the pitched rows and crops them."""
    item = np.dtype(dtype).itemsize * comps
    assert img.texel_bytes == item and img.pitch_bytes % item == 0
    raw = _d2h((np.zeros((img.height, img.pitch_bytes // item, comps), dtype=dtype), img.d_ptr))[0]
    return np.ascontiguousarray(raw[:, :img.width]).reshape(img.width * img.height, comps)


class _Pass:
    """A pass object over its zr_<prefix>_* entry points. A subclass states what differs: its prefix, its params struct
    (Params, when the pass has <prefix>_default_params), whether <prefix>_get_output takes an output id, and its Render
    inputs. A verb the pass does not export raises AttributeError naming the missing entry point."""
    prefix = None
    Params = None
    output_ids = False
    _owned = False

    def __init__(self, w, h):
        self._create(w, h)

    def _create(self, *size):
        self.handle = C.c_void_p()
        check(getattr(lib, self.prefix + "_create")(*size, C.byref(self.handle)))
        self._owned = True
        self._load_default_params()

    @classmethod
    def _borrow(cls, handle):
        """A wrapper over a pass another object owns (a Renderer): this wrapper neither creates nor destroys it."""
        self = cls.__new__(cls)
        self.handle = handle
        self._load_default_params()
        return self

    def _load_default_params(self):
        if self.Params is not None:
            self.params = self.Params()
            check(getattr(lib, self.prefix + "_default_params")(C.byref(self.params)))

    def _call(self, verb, *args):
        check(getattr(lib, self.prefix + "_" + verb)(self.handle, *args))

    def SetParams(self, **kw):
        """Sets the named fields on a copy of `params`; the copy becomes `params` only once the pass has accepted it."""
        p = self.Params.from_buffer_copy(self.params)
        for k, v in kw.items():
            setattr(p, k, v)
        self._call("set_params", C.byref(p))
        self.params = p

    def OnWindowResized(self, w, h):
        self._call("resize", w, h)

    def ResetTemporal(self):
        self._call("reset_temporal")

    def SetRows(self, y0, y1):
        self._call("set_rows", y0, y1)

    def SetHaloExchange(self, fn):
        """fn: a _lib.HALO_EXCHANGE_FN, kept alive here while the pass may call it, or None to remove the hook."""
        self._call("set_halo_exchange", fn, None)
        self._halo_exchange = fn

    def SetReduce(self, fn):
        """fn: a _lib.REDUCE_U32_FN, kept alive here while the pass may call it, or None to remove the hook."""
        self._call("set_reduce", fn, None)
        self._reduce = fn

    def SetCostMap(self, d_cycles):
        """d_cycles: device address of the per-tile uint64 cycle counters, or 0 to stop counting."""
        self._call("set_cost_map", d_cycles)

    def SetScheduleCosts(self, tile_costs, tiles_x, tiles_y):
        """tile_costs: sequence of tiles_x * tiles_y floats (row-major) or None."""
        arr = None if tile_costs is None else (C.c_double * (tiles_x * tiles_y))(*tile_costs)
        self._call("set_schedule_costs", arr, tiles_x, tiles_y)

    def Render(self, fi, stream=None):
        self._call("render", C.byref(fi), stream)

    def GetOutput(self, which=0):
        """The output image; `which` picks one of the zr_*_output planes of a pass that has several."""
        if which and not self.output_ids:
            raise ValueError("%s has a single output" % type(self).__name__)
        img = _lib.Image2D()
        self._call("get_output", *((which,) if self.output_ids else ()), C.byref(img))
        return img

    def __del__(self):
        try:
            if self._owned and self.handle:
                getattr(lib, self.prefix + "_destroy")(self.handle)
                self.handle = None
        except Exception:
            pass


class GBufferRT(_Pass):
    prefix = "zr_gbuffer_pass"
    NO_PICK = 0xffffffff

    def __init__(self):
        self._create()

    def Pick(self, x, y):
        """GBufferRT::PickPixel: the next Render writes the instance index under pixel (x, y) (NO_PICK for none) into the pick word."""
        self._call("pick", int(x), int(y))

    def GetPick(self):
        """The pick word (waits for the default stream): the instance index the last picking Render found, or NO_PICK."""
        img = _lib.Image2D()
        self._call("get_pick", C.byref(img))
        return int(_d2h((np.zeros(1, dtype=np.uint32), img.d_ptr))[0][0])


def _lut_arg(lut):
    """A set_sky argument: the LUT image (a SkyPass's GetOutput()) by reference, or None for off."""
    return None if lut is None else C.byref(lut)


class DirectLighting(_Pass):
    prefix = "zr_direct_pass"
    Params = _lib.DirectParams
    output_ids = True

    def SetSky(self, lut):
        """The sky in accumulating frames: pixels without geometry accumulate Le_SkyWithSunDisk from the sky-view LUT `lut` (a
        SkyPass's GetOutput(), which must outlive its use here); None turns it off."""
        self._call("set_sky", _lut_arg(lut))


class IndirectLighting(_Pass):
    prefix = "zr_indirect_pass"
    Params = _lib.IndirectParams
    output_ids = True
    # zr_rpt_debug_view (RPT_DEBUG_VIEW)
    (DEBUG_VIEW_NONE, DEBUG_VIEW_K, DEBUG_VIEW_CASE, DEBUG_VIEW_FOUND_CONNECTION, DEBUG_VIEW_CONNECTION_LOBE_K_MIN_1,
     DEBUG_VIEW_CONNECTION_LOBE_K) = range(6)

    def SetDebugView(self, view):
        """DebugViewCallback: the indirect output shows each pixel's reconnection (its k, case, whether there is one, or the
        lobe before or after it) instead of radiance; DEBUG_VIEW_NONE returns to radiance."""
        self._call("set_debug_view", int(view))


class IndirectLightingGI(_Pass):
    """IndirectLighting with INTEGRATOR::ReSTIR_GI (zr_gi_pass, csrc/rgi.cu)."""
    prefix = "zr_gi_pass"
    Params = _lib.GIParams
    output_ids = True
    PATH_TRACING, RESTIR_GI = 0, 1

    def SetMethod(self, integrator):
        """IndirectLighting::SetMethod for the two integrators this pass object runs: the plain path tracer
        (PathTracer.hlsl) or ReSTIR GI."""
        self._call("set_method", int(integrator))


class Compositing(_Pass):
    prefix = "zr_compositing_pass"

    def SetParams(self, emissive_di=1, indirect=1, firefly_filter=1):
        self._call("set_params", C.byref(_lib.CompositingParams(emissive_di, indirect, firefly_filter)))

    def Render(self, fi, d_direct, d_indirect, stream=None):
        self._call("render", C.byref(fi), d_direct, d_indirect, stream)

    def SetSky(self, lut):
        """The sky behind geometry in frames that do not accumulate (with emissive_di on), from the sky-view LUT `lut`; None
        turns it off."""
        self._call("set_sky", _lut_arg(lut))


class SkyPass(_Pass):
    """Sky (zr_sky_pass, csrc/sky.cu): the lut_w x lut_h sky-view LUT of the frame's sun and atmosphere, R11G11B10F texels as
    uint32 (GetOutput)."""
    prefix = "zr_sky_pass"

    def Render(self, fi, stream=None):
        self._call("render", C.byref(fi), stream)


class TAA(_Pass):
    prefix = "zr_taa_pass"

    def Render(self, fi, d_signal, stream=None):
        self._call("render", C.byref(fi), d_signal, stream)


class SVGF(_Pass):
    """SVGF denoiser (zr_svgf_pass_*): RGBA32F signal in, RGBA32F out (alpha = filtered variance); between Compositing and TAA."""
    prefix = "zr_svgf_pass"
    Params = _lib.SvgfParams
    output_ids = True

    def Render(self, fi, d_signal, stream=None):
        self._call("render", C.byref(fi), d_signal, stream)


class AutoExposure(_Pass):
    """AutoExposure (zr_auto_exposure_pass, csrc/display.cu): luminance histogram of the TAA input -> adapted exposure.
    GetOutput() is the 1 x 1 float2 {exposure, adapted luminance}; Render reads the frame's dt (seconds)."""
    prefix = "zr_auto_exposure_pass"
    Params = _lib.AutoExposureParams

    def Render(self, fi, d_signal, stream=None):
        self._call("render", C.byref(fi), d_signal, stream)


class Display(_Pass):
    """Display (zr_display_pass, csrc/display.cu): TAA output x exposure -> tone mapper -> sRGB RGBA8."""
    prefix = "zr_display_pass"
    Params = _lib.DisplayParams
    NONE, NEUTRAL, AGX_DEFAULT, AGX_GOLDEN, AGX_PUNCHY, AGX_CUSTOM = range(6)
    # zr_display_view (DisplayOption)
    (VIEW_DEFAULT, VIEW_BASE_COLOR, VIEW_NORMAL, VIEW_METALNESS_ROUGHNESS, VIEW_COAT_WEIGHT, VIEW_COAT_COLOR, VIEW_ROUGHNESS_TH,
     VIEW_EMISSIVE, VIEW_TRANSMISSION, VIEW_DEPTH) = range(10)
    MAX_PICKED = 32

    def SetView(self, view, roughness_th=1.0):
        """DisplayOptionCallback: a G-buffer debug view in place of the tone-mapped image (VIEW_DEFAULT returns to it)."""
        self._call("set_view", int(view), float(roughness_th))

    def SetPicked(self, instances):
        """SetPickedInstance / GetPickedInstances: outline these instance indices (at most MAX_PICKED; empty clears)."""
        a = np.ascontiguousarray(np.asarray(instances, dtype=np.int64).reshape(-1)).astype(np.uint32)
        self._call("set_picked", _vp(a) if len(a) else None, len(a))

    def SetLUT(self, lut):
        """lut: the Tony McMapface LUT as packed R9G9B9E5 texels, uint32[48][48][48] (x fastest)."""
        a = np.ascontiguousarray(lut, dtype=np.uint32)
        self._call("set_lut", _vp(a), a.shape[0] if a.ndim == 3 else 0)

    def Render(self, fi, d_signal, d_exposure, stream=None):
        self._call("render", C.byref(fi), d_signal, d_exposure, stream)


class Comm:
    """zr_comm: halo transport between strips (NCCL, bound inside the library). `Comm.from_torch()` distributes the id through an
    initialised torch.distributed process group; any other out-of-band channel works with Comm.unique_id() / Comm(id, rank, world).
    `Comm.from_transport()` moves the bands with the caller's own functions instead."""

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

    @classmethod
    def from_transport(cls, exchange_halos, gather_rows, allreduce_u32, rank, world):
        """zr_comm_create_transport: three callables taking the arguments of the _lib.CommTransport fields and returning a
        zr_status (0 = OK). An exception cannot cross the C frames that call them: catch it and return an error status.
        The callables stay alive as long as this Comm."""
        self = cls.__new__(cls)
        self.handle, self.rank, self.world = C.c_void_p(), rank, world
        self._transport = _lib.CommTransport(*(ftype(fn) for (_, ftype), fn in zip(_lib.CommTransport._fields_,
                                                                                (exchange_halos, gather_rows, allreduce_u32))))
        check(lib.zr_comm_create_transport(C.byref(self._transport), None, int(rank), int(world), C.byref(self.handle)))
        return self

    def allreduce_u32(self, d_values, n, stream=None, which_comm=0):
        """In-place sum of n uint32 values (device pointer) over every rank."""
        check(lib.zr_comm_allreduce_u32(self.handle, int(which_comm), d_values, n, stream))

    def stats(self):
        b, c = C.c_uint64(), C.c_uint64()
        check(lib.zr_comm_stats(self.handle, C.byref(b), C.byref(c)))
        return b.value, c.value

    def close(self):
        if self.handle:
            lib.zr_comm_destroy(self.handle)
            self.handle = None


class Renderer:
    """The frame driver (zr_renderer, csrc/renderer.cu): G-buffers + all passes, one Render(frame constants) per frame.

    Its passes are reached through one wrapper each (gbuffer, direct, indirect, compositing, taa, and gi, svgf,
    auto_exposure, display once enabled); a pass the renderer keeps across a call keeps its wrapper and its params."""

    def __init__(self, scene, w, h, two_streams=True, with_tridiff=False):
        self.scene = scene
        self.handle = C.c_void_p()
        desc = _lib.RendererDesc(w, h, int(with_tridiff), int(two_streams))
        check(lib.zr_renderer_create(C.byref(desc), scene.handle, C.byref(self.handle)))
        hs = [C.c_void_p() for _ in range(5)]
        check(lib.zr_renderer_get_passes(self.handle, *[C.byref(x) for x in hs]))
        self.gbuffer, self.direct, self.indirect, self.compositing, self.taa = (
            cls._borrow(hnd) for cls, hnd in zip((GBufferRT, DirectLighting, IndirectLighting, Compositing, TAA), hs))
        self.gi = self.svgf = self.auto_exposure = self.display = self.sky = None

    @staticmethod
    def _wrapper(current, cls, handle):
        """`current` while it still wraps the native pass `handle`, else a new wrapper; None when there is no pass."""
        if not handle:
            return None
        return current if current is not None and current.handle.value == handle.value else cls._borrow(handle)

    def Render(self, fc, stream=None):
        check(lib.zr_renderer_render(self.handle, C.byref(fc), stream))

    PATH_TRACING, RESTIR_GI, RESTIR_PT = 0, 1, 2

    def SetMethod(self, integrator):
        """IndirectLighting::SetMethod as the renderer calls it (DefaultRenderer.cpp:243). `gi` is the pass that runs the
        path tracer and ReSTIR GI, None until one of them has been selected."""
        check(lib.zr_renderer_set_integrator(self.handle, int(integrator)))
        h = C.c_void_p()
        check(lib.zr_renderer_get_gi_pass(self.handle, C.byref(h)))
        self.gi = self._wrapper(self.gi, IndirectLightingGI, h)

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
        self.svgf = self._wrapper(self.svgf, SVGF, h)

    def SetDisplay(self, enable=True, lut=None):
        """AutoExposure on the TAA input and Display on the TAA output (PostProcessor.cpp). lut: the Tony McMapface LUT the
        default NEUTRAL tone mapper needs (Display.SetLUT)."""
        ae, disp = C.c_void_p(), C.c_void_p()
        check(lib.zr_renderer_set_display(self.handle, int(enable), C.byref(ae), C.byref(disp)))
        self.auto_exposure = self._wrapper(self.auto_exposure, AutoExposure, ae)
        self.display = self._wrapper(self.display, Display, disp)
        if enable and lut is not None:
            self.display.SetLUT(lut)

    def SetSky(self, enable=True):
        """The sky behind geometry: a 256 x 128 SkyPass recomputed every frame before DirectLighting, read by DirectLighting and
        Compositing. False frees it."""
        h = C.c_void_p()
        check(lib.zr_renderer_set_sky(self.handle, int(enable), C.byref(h)))
        self.sky = self._wrapper(self.sky, SkyPass, h)

    def Pick(self, x, y):
        """DefaultRenderer::Pick: the next Render reports the instance under pixel (x, y) (GBufferRT.Pick)."""
        self.gbuffer.Pick(x, y)

    def GetPick(self):
        """The instance the last picking Render found under its pixel, GBufferRT.NO_PICK for none. In a strip-sharded frame it is
        what this rank's rows show: NO_PICK on a rank whose rows do not hold the pixel."""
        return self.gbuffer.GetPick()

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
