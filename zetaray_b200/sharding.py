"""Strip plans for sharded frames, and the stand-alone-pass frame on one stream.

Strip-sharded frames (SURVEY 8e; the reference is single-GPU) run in the native renderer: zr_renderer_set_shard with a zr_comm
(Renderer.SetShard / Comm in passes.py). A frame is split into horizontal strips whose boundaries are multiples of 32 rows;
StripPlan holds that split. Strips are balanced by measured cost: during the unsharded warm-up frames the lighting kernels
accumulate the SM cycles each 32-row band costs (zr_*_pass_set_cost_map), and StripPlan.balanced() cuts the prefix sum evenly.

ShardedFrame runs the same frame as the renderer from the stand-alone pass objects on ONE stream, for a whole image on one GPU:
each kernel's timing events then cover only that kernel, and the G-buffers stay reachable for download."""
import ctypes as C

UNIT = 32       # strip granularity in rows == sort tile == halo
HALO = 32


class StripPlan:
    """bounds[r] .. bounds[r + 1] = rows of rank r; every bound except the last is a multiple of UNIT."""

    def __init__(self, height, bounds):
        self.height = int(height)
        self.bounds = [int(b) for b in bounds]
        assert self.bounds[0] == 0 and self.bounds[-1] == self.height
        for a, b in zip(self.bounds, self.bounds[1:]):
            assert b > a, "every rank needs at least one band"
        for b in self.bounds[1:-1]:
            assert b % UNIT == 0

    @property
    def world(self):
        return len(self.bounds) - 1

    def rows(self, rank):
        return self.bounds[rank], self.bounds[rank + 1]

    def rows_with_halo(self, rank, halo=HALO):
        y0, y1 = self.rows(rank)
        return max(0, y0 - halo), min(self.height, y1 + halo)

    @staticmethod
    def num_units(height):
        return (height + UNIT - 1) // UNIT

    @classmethod
    def uniform(cls, height, world):
        return cls.balanced(height, world, [1.0] * cls.num_units(height))

    @classmethod
    def balanced(cls, height, world, unit_costs):
        """Contiguous partition of the 32-row bands into `world` strips minimising the largest strip cost
        (exact: binary search on the bottleneck + greedy feasibility; n <= a few hundred bands)."""
        n = cls.num_units(height)
        costs = [max(float(c), 0.0) for c in unit_costs]
        assert len(costs) == n and 1 <= world <= n
        if world == 1:
            return cls(height, [0, height])
        eps = 1e-9 * (sum(costs) + 1.0)
        costs = [c + eps for c in costs]      # zero-cost bands (sky) still have to belong to somebody

        def cuts_for(limit):
            cuts, acc = [0], 0.0
            for i, c in enumerate(costs):
                if acc > 0 and acc + c > limit * (1 + 1e-12):     # greedy: close the strip when the next band would overflow it
                    cuts.append(i)
                    acc = 0.0
                acc += c
            cuts.append(n)
            return cuts

        lo, hi = max(costs), sum(costs) * (1 + 1e-9)
        for _ in range(60):
            mid = 0.5 * (lo + hi)
            if len(cuts_for(mid)) - 1 <= world:
                hi = mid
            else:
                lo = mid
        cuts = cuts_for(hi)
        # fewer strips than ranks: split the widest strips until every rank owns at least one band
        while len(cuts) - 1 < world:
            widths = [(cuts[i + 1] - cuts[i], i) for i in range(len(cuts) - 1)]
            w, i = max(widths)
            assert w >= 2
            seg = costs[cuts[i]:cuts[i + 1]]
            half, acc, k = 0.5 * sum(seg), 0.0, 1
            for j, c in enumerate(seg[:-1]):
                acc += c
                k = j + 1
                if acc >= half:
                    break
            cuts.insert(i + 1, cuts[i] + k)
        bounds = [min(c * UNIT, height) for c in cuts]
        bounds[-1] = height
        return cls(height, bounds)

    def strip_costs(self, unit_costs):
        return [sum(unit_costs[a // UNIT:(b + UNIT - 1) // UNIT]) for a, b in zip(self.bounds, self.bounds[1:])]


class ShardedFrame:
    """GBufferRT -> DirectLighting -> IndirectLighting -> Compositing -> TAA on one stream, the whole image.

    passes: dict(gbuffer=GBufferRT, direct=DirectLighting, indirect=IndirectLighting, compositing=Compositing, taa=TAA)"""

    def __init__(self, passes, gbuffers, width, height, rank, world):
        if world != 1:
            raise ValueError("ShardedFrame renders the whole frame on one GPU; strip-sharded frames run in the native "
                             "renderer (Renderer.SetShard)")
        self.p, self.gb = passes, gbuffers
        self.W, self.H = width, height

    def render(self, fi, fc, stream):
        """One frame on `stream` (a torch.cuda.Stream)."""
        p = self.p
        st = C.c_void_p(stream.cuda_stream)
        self.gb.flip()
        fi.frame = fc
        self.gb.fill_inputs(fi)
        p["gbuffer"].Render(fi, st)
        p["direct"].Render(fi, st)
        p["indirect"].Render(fi, st)
        p["compositing"].Render(fi, p["direct"].GetOutput(0).d_ptr, p["indirect"].GetOutput(0).d_ptr, st)
        p["taa"].Render(fi, p["compositing"].GetOutput().d_ptr, st)
