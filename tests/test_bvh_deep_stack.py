"""CPU tier: the traversal's node-group stack past its register-resident entries (zr_scene.cuh::Traverse keeps the top
BVH_STACK_REGS entries in registers and spills deeper ones to a local array). The benchmark scenes are too shallow to reach the
spill path on every run, so this test builds a tree deep enough by construction and sends rays that must walk all of it."""
import os
import re

import numpy as np

from tests import hostsim
from tests.orc import ptr
from tests.test_bvh_host import build, make_rays, THREADS

HEADER = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "zetaray_b200", "csrc", "zr_bvh.h")


def stack_regs():
    with open(HEADER) as f:
        return int(re.search(r"#define ZR_BVH_STACK_REGS (\d+)", f.read()).group(1))


def line_scene(n):
    """n right triangles in the plane z = 0, strung along x with cubic spacing (dense near x = 0, so the SAH tree is deep there), and
    one wall across the line's far end. A ray along x inside the plane passes through every child box of the tree and hits no
    triangle of the line (it is parallel to them); going +x it ends on the wall."""
    wt = np.zeros((n + 1, 9), dtype=np.float32)
    wt[:n, 0] = np.arange(n, dtype=np.float64) ** 3 / n ** 2
    wt[:n, 3] = 0.5; wt[:n, 7] = 1.0          # e1 = (0.5, 0, 0), e2 = (0, 1, 0)
    x_end = float(wt[n - 1, 0]) + 2.0
    wt[n, 0:3] = (x_end, -1.0, -1.0); wt[n, 3:6] = (0.0, 4.0, 0.0); wt[n, 6:9] = (0.0, 0.0, 4.0)
    return wt, x_end


def test_traversal_past_the_register_resident_stack():
    hs = hostsim.load()
    wt, x_end = line_scene(4096)
    nodes, order, leaf, (num_nodes, num_tris, max_depth, _) = build(wt)
    # a tree of depth D needs D - 1 stack entries; more than the registers hold, so the deep part of the stack is used
    assert max_depth - 1 > stack_regs(), (max_depth, stack_regs())
    assert max_depth == 8
    n = num_tris                # the wall is the last one
    tri_mesh = np.zeros(n, dtype=np.uint32)
    first = np.zeros(1, dtype=np.uint32)
    ys = (0.125, 0.25, 0.5, 0.75)
    walk = np.zeros((2 * len(ys), 8), dtype=np.float32)
    for i, y in enumerate(ys):
        walk[i] = (-1.0, y, 0.0, 0.0, 1.0, 0.0, 0.0, 3.0e38)             # +x: through every box, onto the wall
        walk[len(ys) + i] = (x_end - 1.0, y, 0.0, 0.0, -1.0, 0.0, 0.0, 3.0e38)   # -x from beyond the line: hits nothing
    rays = np.concatenate([walk, make_rays(wt, 2000, 5, np.array((-5.0, 0.5, 0.3), dtype=np.float32))])
    got = np.zeros((len(rays), 4), dtype=np.float32)
    anyf = np.zeros(len(rays), dtype=np.uint32)
    hs.hostsim_trace(ptr(nodes), ptr(leaf), ptr(tri_mesh), ptr(first), ptr(rays), len(rays), ptr(got), ptr(anyf), None, THREADS)
    ref = np.zeros((len(rays), 4), dtype=np.float32)
    hs.hostsim_brute(ptr(wt), n, ptr(rays), len(rays), ptr(ref), THREADS)
    assert got.tobytes() == ref.tobytes(), int((got.view(np.uint32) != ref.view(np.uint32)).any(axis=1).sum())
    hit = ref[:, 0] < 3.0e38
    assert np.array_equal(anyf != 0, hit)
    assert hit[:len(ys)].all() and (ref[:len(ys), 3].view(np.uint32) == n - 1).all() and not hit[len(ys):len(walk)].any()
    # the walking rays visit every node once: no stack entry was lost on the way down or back up
    for anyhit, sel in ((0, slice(0, len(walk))), (1, slice(len(ys), len(walk)))):
        visits = np.zeros(len(walk), dtype=np.uint32); tests = np.zeros(len(walk), dtype=np.uint32)
        hs.hostsim_trace_stats(ptr(nodes), ptr(leaf), ptr(tri_mesh), ptr(first), ptr(walk), len(walk), ptr(visits), ptr(tests), anyhit)
        assert (visits[sel] == num_nodes).all(), (anyhit, visits, num_nodes)
