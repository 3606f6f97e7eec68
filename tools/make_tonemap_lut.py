"""Converts the Tony McMapface tone-mapping LUT of the reference (Assets/LUT/tony_mc_mapface.dds) into the test fixture
tests/golden/tony_mc_mapface.npz: the raw R9G9B9E5_SHAREDEXP texels as uint32[48][48][48] (z, y, x; x fastest, as the DDS
stores them) and the sha256 of that payload. Needs a ZetaRay checkout; the committed fixture is what the tests read.

    python tools/make_tonemap_lut.py path/to/ZetaRay"""
import hashlib
import os
import struct
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DXGI_FORMAT_R9G9B9E5_SHAREDEXP = 67
DIM = 48


def read_dds_rgb9e5(path):
    raw = open(path, "rb").read()
    if raw[:4] != b"DDS ":
        raise ValueError("%s: not a DDS file" % path)
    size, flags, height, width, pitch, depth = struct.unpack_from("<6I", raw, 4)
    fourcc = raw[84:88]
    if size != 124 or fourcc != b"DX10":
        raise ValueError("%s: expected a DX10 extended header" % path)
    dxgi_format, dimension, misc, array_size, misc2 = struct.unpack_from("<5I", raw, 128)
    if dxgi_format != DXGI_FORMAT_R9G9B9E5_SHAREDEXP or dimension != 4:        # 4 = D3D10_RESOURCE_DIMENSION_TEXTURE3D
        raise ValueError("%s: format %d / dimension %d, expected R9G9B9E5 3D" % (path, dxgi_format, dimension))
    if (width, height, depth) != (DIM, DIM, DIM):
        raise ValueError("%s: %dx%dx%d, expected %d^3" % (path, width, height, depth, DIM))
    payload = raw[148:148 + DIM ** 3 * 4]
    if len(payload) != DIM ** 3 * 4:
        raise ValueError("%s: truncated payload" % path)
    return np.frombuffer(payload, dtype="<u4").reshape(DIM, DIM, DIM).copy(), hashlib.sha256(payload).hexdigest()


def main():
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    ref = sys.argv[1]
    lut, digest = read_dds_rgb9e5(os.path.join(ref, "Assets", "LUT", "tony_mc_mapface.dds"))
    out = os.path.join(ROOT, "tests", "golden", "tony_mc_mapface.npz")
    np.savez_compressed(out, lut=lut, sha256=np.array(digest))
    print("wrote", out, lut.shape, digest)


if __name__ == "__main__":
    main()
