"""The default camera of the reference and its per-frame constants (cbFrameConstants) for headless runs: bench.py, smoke and the
tests all render with this producer (SURVEY 8a-19; the reference's is Common::UpdateFrameConstants, DefaultRenderer.cpp:31-125)."""
import numpy as np

from ._lib import FrameConstants


def look_at_frame_constants(w, h, frame=1, jitter=(0.0, 0.0), prev_jitter=(0.0, 0.0), cam=(0.0, 1.2, -4.043), prev_cam=None):
    """cbFrameConstants for the default camera (SURVEY 8a-19): left-handed, +Z forward, vfov 60 deg.
    prev_cam: last frame's camera position (a translating camera); defaults to cam (static)."""
    fc = FrameConstants()
    pc = cam if prev_cam is None else prev_cam
    view = np.array([[1, 0, 0, -cam[0]], [0, 1, 0, -cam[1]], [0, 0, 1, -cam[2]]], dtype=np.float32)
    inv = np.array([[1, 0, 0, cam[0]], [0, 1, 0, cam[1]], [0, 0, 1, cam[2]]], dtype=np.float32)
    pview = np.array([[1, 0, 0, -pc[0]], [0, 1, 0, -pc[1]], [0, 0, 1, -pc[2]]], dtype=np.float32)
    pinv = np.array([[1, 0, 0, pc[0]], [0, 1, 0, pc[1]], [0, 0, 1, pc[2]]], dtype=np.float32)
    for name, m in (("CurrView", view), ("PrevView", pview), ("CurrViewInv", inv), ("PrevViewInv", pinv)):
        arr = getattr(fc, name)
        for i, v in enumerate(m.reshape(-1)):
            arr[i] = float(v)
    fc.CameraPos[0], fc.CameraPos[1], fc.CameraPos[2] = cam
    fc.CameraNear = 0.2
    fc.AspectRatio = np.float32(w) / np.float32(h)
    fc.TanHalfFOV = float(np.tan(np.float32(0.5) * np.float32(np.pi / 3)).astype(np.float32))
    fc.PixelSpreadAngle = float(np.arctan(np.float32(2 * fc.TanHalfFOV / h)))
    fc.FrameNum = frame
    fc.RenderWidth, fc.RenderHeight, fc.DisplayWidth, fc.DisplayHeight = w, h, w, h
    fc.CurrCameraJitter[0], fc.CurrCameraJitter[1] = jitter
    fc.PrevCameraJitter[0], fc.PrevCameraJitter[1] = prev_jitter
    fc.CameraRayUVGradsScale = 1.0
    fc.NumFramesCameraStatic = 0
    fc.CameraStatic = 0
    fc.Accumulate = 0
    set_default_atmosphere(fc)
    return fc


def set_default_atmosphere(fc):
    """The reference's sun and atmosphere (DefaultRenderer.cpp:274-307 with DefaultRendererImpl.h:29-36): distances in km, Hillaire's
    (2020) Rayleigh / Mie / ozone coefficients in 1/km, Rayleigh and ozone stored as a unit colour times a scale. Only the sky
    (zr_renderer_set_sky) reads these fields."""
    f = np.float32
    sun = np.array([0.6565358, -0.0560669, 0.752208233], dtype=np.float64)
    sun = (sun / np.linalg.norm(sun)).astype(np.float32)
    fc.SunDir[0], fc.SunDir[1], fc.SunDir[2] = (float(v) for v in sun)
    fc.SunIlluminance = 20.0
    cos_r = f(np.cos(np.float64(np.radians(f(0.5) * f(0.526)))))
    fc.SunCosAngularRadius = float(cos_r)
    fc.SunSinAngularRadius = float(np.sqrt(f(1.0) - cos_r * cos_r))
    fc.AtmosphereAltitude = 100.0
    fc.PlanetRadius = 6360.0
    fc.g = 0.8
    for name, v in (("RayleighSigmaS", (5.802e-3, 13.558e-3, 33.1e-3)), ("OzoneSigmaA", (0.65e-3, 1.881e-3, 0.085e-3))):
        v = np.array(v, dtype=np.float32)
        scale = f(np.sqrt(np.float64(v @ v)))
        color = v * (f(1.0) / scale)
        arr = getattr(fc, name + "Color")
        arr[0], arr[1], arr[2] = (float(c) for c in color)
        setattr(fc, name + "Scale", float(scale))
    fc.MieSigmaA = 4.4e-3
    fc.MieSigmaS = 3.996e-3



def halton(i, b):
    f = np.float32(1.0); r = np.float32(0.0); bf = np.float32(b)
    while i > 0:
        f = np.float32(f / bf)
        r = np.float32(r + f * np.float32(i % b))
        i = int(np.float32(i) / bf)
    return r


class FrameSequence:
    """cbFrameConstants for consecutive frames of a static camera (SURVEY 8a-19): jitter = Halton(2,3) - 0.5
    over an 8-phase cycle, prev* = last frame's curr*."""

    def __init__(self, w, h, jitter=True, first_frame=1, cam_path=None, accumulate=False):
        """cam_path(frame) -> camera position (a translating camera); None = the static default camera.
        accumulate: Accumulate + CameraStatic with NumFramesCameraStatic counting up (the reference's accumulation mode)."""
        self.w, self.h, self.jitter = w, h, jitter
        self.frame = first_frame - 1
        self.prev_jitter = (0.0, 0.0)
        self.cam_path, self.accumulate = cam_path, accumulate
        self.prev_cam = None
        self.static_frames = 0
        self.scene_changed_pending = False

    def next(self):
        self.frame += 1
        j = (0.0, 0.0)
        if self.jitter:
            ph = self.frame % 8
            j = (float(halton(ph + 1, 2) - np.float32(0.5)), float(halton(ph + 1, 3) - np.float32(0.5)))
        if self.cam_path is None:
            fc = look_at_frame_constants(self.w, self.h, frame=self.frame, jitter=j, prev_jitter=self.prev_jitter)
        else:
            cam = tuple(float(np.float32(c)) for c in self.cam_path(self.frame))
            fc = look_at_frame_constants(self.w, self.h, frame=self.frame, jitter=j, prev_jitter=self.prev_jitter, cam=cam,
                                               prev_cam=self.prev_cam or cam)
            self.prev_cam = cam
        if self.accumulate:
            if self.scene_changed_pending:
                self.static_frames = 0
                fc.Accumulate, fc.CameraStatic, fc.NumFramesCameraStatic = 1, 0, 0
            else:
                self.static_frames += 1
                fc.Accumulate, fc.CameraStatic, fc.NumFramesCameraStatic = 1, 1, self.static_frames
        self.scene_changed_pending = False
        self.prev_jitter = j
        return fc

    def scene_changed(self):
        """DefaultRenderer::SceneModified (DefaultRenderer.cpp:96-102, 553-556): the next frame says CameraStatic = 0 and
        NumFramesCameraStatic = 0, so accumulation starts over from the frame after it. Call it after an edit such as
        Scene.update_materials."""
        self.scene_changed_pending = True
