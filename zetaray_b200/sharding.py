"""Strip-sharded frames across GPUs (SURVEY 8e; the reference is single-GPU, so this has no counterpart there).

One process per GPU. A frame is split into horizontal strips whose boundaries are multiples of 32 rows; every
pass renders only its strip (zr_*_pass_set_rows) and reads up to HALO = 32 rows beyond it. Rows another strip
reads are made coherent at four exchange points per frame (one grouped NCCL send/recv between neighbouring strips, or
-- `halo_mode="allgather"` -- ONE all-gather, the scheme BASELINE.json names):

    after ReSTIR DI temporal      32 B/px reservoirs          (hook called by zr_direct_pass_render)
    after ReSTIR PT temporal      64 B/px reservoirs          (hook called by zr_indirect_pass_render)
    after each PT spatial pass    64 B/px reservoirs          (same hook; they are next frame's "previous")
    before Compositing            DI + indirect finals, 2 x 16 B/px, and the TAA history, 8 B/px

Each rank contributes the top and the bottom HALO rows of its own strip; after the gather it copies its upper
neighbour's bottom band and its lower neighbour's top band into its own full-size planes. Nothing else moves:
the G-buffer halo is re-rendered locally, and scene / BVH / alias table are replicated.

Strips are balanced by measured cost: during the (unsharded) warm-up frames the lighting kernels accumulate the
SM cycles each 32-row band costs (zr_*_pass_set_cost_map); StripPlan.balanced() cuts the prefix sum evenly.

The planning and packing logic is backend-agnostic (torch tensors + torch.distributed), so the same code runs
under gloo on CPU tensors in tests/test_sharding.py."""
import ctypes as C

import torch
import torch.distributed as dist

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


def _band_rows(plan, rank):
    """(top band, bottom band) row ranges of a rank's own strip; each at most HALO rows."""
    y0, y1 = plan.rows(rank)
    return (y0, min(y0 + HALO, y1)), (max(y1 - HALO, y0), y1)


class HaloExchanger:
    """Makes the boundary bands of row-major planes coherent between neighbouring strips. A plane is a uint8 tensor of
    shape [H, pitch_bytes]. Two transports with identical results:

    "p2p" (default)   every rank sends its top band to the rank above and its bottom band to the rank below, straight out
                      of / into the planes (a band is a contiguous row range, so nothing is packed or unpacked); one
                      grouped NCCL send/recv per exchange. Traffic per rank is independent of the number of GPUs.
    "allgather"       the scheme named in BASELINE.json: every rank contributes both bands to ONE all-gather and copies its
                      two neighbours' bands out of the result. Traffic grows with the number of GPUs."""

    def __init__(self, plan, rank, group=None, mode="p2p"):
        assert mode in ("p2p", "allgather")
        self.plan, self.rank, self.group, self.mode = plan, rank, group, mode
        self.world = plan.world
        self._bufs = {}
        self.bytes_sent = 0
        self.calls = 0

    def _buffers(self, nbytes, like):
        key = (nbytes, like.device)
        if key not in self._bufs:
            self._bufs[key] = (torch.empty(nbytes, dtype=torch.uint8, device=like.device),
                               torch.empty(self.world * nbytes, dtype=torch.uint8, device=like.device))
        return self._bufs[key]

    def _exchange_p2p(self, planes):
        plan, r = self.plan, self.rank
        (t0, t1), (b0, b1) = _band_rows(plan, r)
        ops = []
        for p in planes:
            if r > 0:
                (_, _), (nb0, nb1) = _band_rows(plan, r - 1)
                ops.append(dist.P2POp(dist.isend, p[t0:t1].reshape(-1), r - 1, self.group))
                ops.append(dist.P2POp(dist.irecv, p[nb0:nb1].reshape(-1), r - 1, self.group))
                self.bytes_sent += (t1 - t0) * p.shape[1]
            if r < self.world - 1:
                (nt0, nt1), (_, _) = _band_rows(plan, r + 1)
                ops.append(dist.P2POp(dist.isend, p[b0:b1].reshape(-1), r + 1, self.group))
                ops.append(dist.P2POp(dist.irecv, p[nt0:nt1].reshape(-1), r + 1, self.group))
                self.bytes_sent += (b1 - b0) * p.shape[1]
        for req in dist.batch_isend_irecv(ops):
            req.wait()
        self.calls += 1

    def exchange(self, planes):
        if self.world == 1:
            return
        if self.mode == "p2p":
            return self._exchange_p2p(planes)
        plan, r = self.plan, self.rank
        slot = [HALO * p.shape[1] for p in planes]            # bytes of one band slot per plane
        packet = 2 * sum(slot)
        send, recv = self._buffers(packet, planes[0])
        (t0, t1), (b0, b1) = _band_rows(plan, r)
        off = 0
        for p, sb in zip(planes, slot):
            pitch = p.shape[1]
            send[off:off + (t1 - t0) * pitch].copy_(p[t0:t1].reshape(-1))
            send[off + sb:off + sb + (b1 - b0) * pitch].copy_(p[b0:b1].reshape(-1))
            off += 2 * sb
        try:
            dist.all_gather_into_tensor(recv, send, group=self.group)
        except (RuntimeError, NotImplementedError):
            parts = [recv[i * packet:(i + 1) * packet] for i in range(self.world)]
            dist.all_gather(parts, send, group=self.group)
        self.bytes_sent += packet
        self.calls += 1
        y0, y1 = plan.rows(r)
        off = 0
        for p, sb in zip(planes, slot):
            pitch = p.shape[1]
            if r > 0:                                          # upper neighbour's bottom band -> rows just above my strip
                (_, _), (nb0, nb1) = _band_rows(plan, r - 1)
                src = recv[(r - 1) * packet + off + sb:(r - 1) * packet + off + sb + (nb1 - nb0) * pitch]
                p[nb0:nb1].reshape(-1).copy_(src)
            if r < self.world - 1:                             # lower neighbour's top band -> rows just below my strip
                (nt0, nt1), (_, _) = _band_rows(plan, r + 1)
                src = recv[(r + 1) * packet + off:(r + 1) * packet + off + (nt1 - nt0) * pitch]
                p[nt0:nt1].reshape(-1).copy_(src)
            off += 2 * sb

    def gather_rows(self, plane, dst_rank=None):
        """Collect every rank's own strip of `plane` (all ranks end up with the full plane; strips are padded to the
        tallest one for the gather)."""
        if self.world == 1:
            return
        plan, r = self.plan, self.rank
        pitch = plane.shape[1]
        tallest = max(b - a for a, b in zip(plan.bounds, plan.bounds[1:]))
        send, recv = self._buffers(tallest * pitch, plane)
        y0, y1 = plan.rows(r)
        send[:(y1 - y0) * pitch].copy_(plane[y0:y1].reshape(-1))
        try:
            dist.all_gather_into_tensor(recv, send, group=self.group)
        except (RuntimeError, NotImplementedError):
            dist.all_gather([recv[i * tallest * pitch:(i + 1) * tallest * pitch] for i in range(self.world)], send, group=self.group)
        for q in range(self.world):
            if q == r:
                continue
            a, b = plan.rows(q)
            plane[a:b].reshape(-1).copy_(recv[q * tallest * pitch:q * tallest * pitch + (b - a) * pitch])


class _DevicePlane:
    """Lets torch wrap a raw device pointer (zr_image2d) without copying."""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes,), "typestr": "|u1", "data": (int(ptr), False), "version": 2}


def plane_tensor(img):
    """uint8 [H, pitch] view of a zr_image2d living on the current CUDA device."""
    nbytes = img.height * img.pitch_bytes
    return torch.as_tensor(_DevicePlane(img.d_ptr, nbytes), device="cuda").view(img.height, img.pitch_bytes)


class ShardedFrame:
    """Runs the frame of bench.py / smoke on this rank's strip and performs the exchanges listed in the module doc.

    passes: dict(gbuffer=GBufferRT, direct=DirectLighting, indirect=IndirectLighting, compositing=Compositing, taa=TAA)"""

    def __init__(self, passes, gbuffers, width, height, rank, world, group=None):
        from . import _lib
        self.p, self.gb = passes, gbuffers
        self.W, self.H, self.rank, self.world = width, height, rank, world
        self.group = group
        self.plan = StripPlan(height, [0, height]) if world == 1 else None
        self.halo = None
        self.tiles_x, self.tiles_y = (width + UNIT - 1) // UNIT, StripPlan.num_units(height)
        self.cost = torch.zeros(self.tiles_x * self.tiles_y, dtype=torch.int64, device="cuda")
        self._hook = _lib.HALO_EXCHANGE_FN(self._on_exchange)
        self._lib = _lib
        self._streams = {}
        self._hook_error = None
        self._events = (torch.cuda.Event(), torch.cuda.Event())

    # ---- cost measurement during unsharded warm-up ----
    def begin_cost_measurement(self):
        self.cost.zero_()
        self.p["direct"].SetCostMap(self.cost.data_ptr())
        self.p["indirect"].SetCostMap(self.cost.data_ptr())

    def end_cost_measurement(self, schedule=False):
        """Returns the cost of every 32-row band (for StripPlan.balanced). With schedule=True the per-tile costs also
        become the lighting passes' block schedule (expensive tiles first; no gain over plain order was seen, the compact per-strip grid is what matters)."""
        self.p["direct"].SetCostMap(0)
        self.p["indirect"].SetCostMap(0)
        c = self.cost.to(torch.float64)
        if self.world > 1:
            dist.all_reduce(c, op=dist.ReduceOp.SUM, group=self.group)     # identical plan on every rank
        tiles = [float(v) for v in c.tolist()]
        if schedule:
            self.p["direct"].SetScheduleCosts(tiles, self.tiles_x, self.tiles_y)
            self.p["indirect"].SetScheduleCosts(tiles, self.tiles_x, self.tiles_y)
        return [sum(tiles[b * self.tiles_x:(b + 1) * self.tiles_x]) for b in range(self.tiles_y)]

    # ---- sharding ----
    def shard(self, plan, halo_mode="p2p"):
        self.plan = plan
        self.halo = HaloExchanger(plan, self.rank, self.group, mode=halo_mode)
        y0, y1 = plan.rows(self.rank)
        g0, g1 = plan.rows_with_halo(self.rank)
        self.p["gbuffer"].SetRows(g0, g1)
        self.p["direct"].SetRows(y0, y1)
        self.p["indirect"].SetRows(y0, y1)
        # the TAA neighbourhood reads the composited signal one row beyond the strip
        self.p["compositing"].SetRows(max(0, y0 - 1), min(self.H, y1 + 1))
        self.p["taa"].SetRows(y0, y1)
        if plan.world > 1:
            self.p["direct"].SetHaloExchange(self._hook)
            self.p["indirect"].SetHaloExchange(self._hook)

    def _on_exchange(self, user, planes, n, stream):
        # called from inside zr_*_pass_render through ctypes: an exception cannot propagate through the C frames, so it
        # is parked here and re-raised by render()
        try:
            tensors = [plane_tensor(planes[i]) for i in range(n)]
            # the torch Stream OBJECT render() was given for this handle: torch ops issued under it are ordered with
            # the kernels the pass launched on the raw handle (wrapping the handle again, in particular handle 0 --
            # the legacy default stream -- in an ExternalStream was observed NOT to give that ordering)
            ts = self._streams.get(int(stream or 0))
            if ts is None:
                raise RuntimeError("halo exchange requested on a stream render() was not given (0x%x)" % int(stream or 0))
            with torch.cuda.stream(ts):
                self.halo.exchange(tensors)
        except BaseException as e:      # noqa: BLE001
            self._hook_error = e

    def _raise_hook_error(self):
        e, self._hook_error = getattr(self, "_hook_error", None), None
        if e is not None:
            raise RuntimeError("halo exchange failed inside a pass") from e

    def render(self, fi, fc, stream, st=None, side=None, st_side=None, ev_g=None, ev_d=None):
        """One frame on `stream` (a torch.cuda.Stream created by the caller -- not the legacy default stream when the
        frame is sharded); `side`: optional second torch stream DirectLighting is recorded on."""
        p = self.p
        if self.halo is not None and self.world > 1 and int(stream.cuda_stream) == 0:
            raise ValueError("a sharded frame needs an explicit torch.cuda.Stream(), not the legacy default stream")
        st = C.c_void_p(stream.cuda_stream)
        self._streams[int(stream.cuda_stream)] = stream
        if side is not None:
            st_side = C.c_void_p(side.cuda_stream)
            self._streams[int(side.cuda_stream)] = side
            if ev_g is None:
                ev_g, ev_d = self._events
        self.gb.flip()
        fi.frame = fc
        self.gb.fill_inputs(fi)
        p["gbuffer"].Render(fi, st)
        if side is not None:
            ev_g.record(stream)
            side.wait_event(ev_g)
            p["direct"].Render(fi, st_side)
        else:
            p["direct"].Render(fi, st)
        p["indirect"].Render(fi, st)
        self._raise_hook_error()
        if side is not None:
            ev_d.record(side)
            stream.wait_event(ev_d)
        if self.halo is not None and self.world > 1:
            with torch.cuda.stream(stream):
                self.halo.exchange([plane_tensor(p["direct"].GetOutput(0)), plane_tensor(p["indirect"].GetOutput(0)),
                                    plane_tensor(p["taa"].GetOutput())])
        p["compositing"].Render(fi, p["direct"].GetOutput(0).d_ptr, p["indirect"].GetOutput(0).d_ptr, st)
        p["taa"].Render(fi, p["compositing"].GetOutput().d_ptr, st)

    def gather_output(self, stream):
        """Full TAA image on every rank (8 B/px strips)."""
        if self.halo is not None and self.world > 1:
            with torch.cuda.stream(stream):
                self.halo.gather_rows(plane_tensor(self.p["taa"].GetOutput()))
