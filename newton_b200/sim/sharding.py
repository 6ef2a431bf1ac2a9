"""World-range sharding of a Model across ranks (SURVEY.md §8(e)).

Worlds are independent (reference ``geometry/broad_phase_common.py:263-268`` rejects cross-world
pairs; ``sim/builder.py:12921-13021`` emits contact pairs per world) and every entity array is
stored world-contiguous (``*_world_start``: reference ``sim/model.py:1081,1180,883``), so rank ``r``
of ``G`` owns worlds ``[r*W/G, (r+1)*W/G)`` as pure slices plus an index rebase.  World ``-1``
shapes (e.g. the ground plane) are static and replicated on every rank.
"""

from __future__ import annotations

import numpy as np
import torch

from .model import _BODY_FIELDS, _COORD_FIELDS, _DOF_FIELDS, _JOINT_FIELDS, _SHAPE_FIELDS, Model


def world_range(world_count: int, rank: int, world_size: int) -> tuple[int, int]:
    if world_count % world_size != 0:
        raise ValueError(f"world_count={world_count} is not divisible by world_size={world_size}")
    per = world_count // world_size
    return rank * per, (rank + 1) * per


def shard_model(model: Model, rank: int, world_size: int) -> Model:
    w0, w1 = world_range(model.world_count, rank, world_size)
    bws = model.numpy("body_world_start")
    jws = model.numpy("joint_world_start")
    sws = model.numpy("shape_world_start")
    aws = model.numpy("articulation_world_start")
    dws = model.numpy("joint_dof_world_start")
    cws = model.numpy("joint_coord_world_start")
    if bws[0] != 0 or bws[-1] != bws[-2] or jws[0] != 0 or jws[-1] != jws[-2]:
        raise NotImplementedError("sharding requires that only shapes live in the global world (-1)")
    if sws[0] != 0:
        raise NotImplementedError("sharding requires global shapes to be stored at the tail")
    b0, b1 = int(bws[w0]), int(bws[w1])
    j0, j1 = int(jws[w0]), int(jws[w1])
    s0, s1 = int(sws[w0]), int(sws[w1])
    a0, a1 = int(aws[w0]), int(aws[w1])
    d0, d1 = int(dws[w0]), int(dws[w1])
    c0, c1 = int(cws[w0]), int(cws[w1])
    g0, g1 = int(sws[-2]), int(sws[-1])  # global tail shapes
    n_local_shapes = s1 - s0
    out = Model(model.device)
    out.world_count = w1 - w0
    out.up_axis = model.up_axis
    out.use_coord_layout_targets = model.use_coord_layout_targets
    out.body_count, out.joint_count = b1 - b0, j1 - j0
    out.shape_count = n_local_shapes + (g1 - g0)
    out.joint_dof_count, out.joint_coord_count = d1 - d0, c1 - c0
    out.articulation_count = a1 - a0
    out.max_joints_per_articulation = model.max_joints_per_articulation
    out.max_dofs_per_articulation = model.max_dofs_per_articulation
    out.body_label = model.body_label[b0:b1]
    out.joint_label = model.joint_label[j0:j1]
    # host-side metadata that ArticulationView needs on a shard (labels, body -> shapes, excluded pairs), re-indexed like the arrays
    out.articulation_label = list(getattr(model, "articulation_label", [])[a0:a1])
    shape_label = getattr(model, "shape_label", [])
    out.shape_label = list(shape_label[s0:s1]) + list(shape_label[g0:g1])

    def shape_id(s):  # model shape index -> shard shape index, None when the shape is not on this shard
        if s0 <= s < s1:
            return s - s0
        if g0 <= s < g1:
            return s - g0 + n_local_shapes
        return None

    out.body_shapes = {-1: [shape_id(s) for s in getattr(model, "body_shapes", {}).get(-1, []) if shape_id(s) is not None]}
    for b in range(b0, b1):
        out.body_shapes[b - b0] = [shape_id(s) for s in getattr(model, "body_shapes", {}).get(b, []) if shape_id(s) is not None]
    out.shape_collision_filter_pairs = {(shape_id(a), shape_id(b)) for a, b in getattr(model, "shape_collision_filter_pairs", ())
                                        if shape_id(a) is not None and shape_id(b) is not None}

    def cut(name, lo, hi):
        return getattr(model, name)[lo:hi].clone()

    for n in _BODY_FIELDS:
        setattr(out, n, cut(n, b0, b1))
    for n in _JOINT_FIELDS:
        setattr(out, n, cut(n, j0, j1))
    for n in _DOF_FIELDS:
        setattr(out, n, cut(n, d0, d1))
    for n in _COORD_FIELDS:
        setattr(out, n, cut(n, c0, c1))
    out.joint_target_q = cut("joint_target_q", c0, c1)
    for n in _SHAPE_FIELDS:
        setattr(out, n, torch.cat([cut(n, s0, s1), cut(n, g0, g1)]))
    out.hull_points = None if model.hull_points is None else model.hull_points.clone()  # the convex-hull vertex pool is shared: shape_hull_start keeps indexing it
    src = getattr(model, "shape_source", None) or [None] * model.shape_count
    out.shape_source = list(src[s0:s1]) + list(src[g0:g1])

    def rebase(t, off):
        return torch.where(t >= 0, t - off, t)

    out.body_world = rebase(out.body_world, w0)
    out.joint_world = rebase(out.joint_world, w0)
    out.shape_world = rebase(out.shape_world, w0)
    out.joint_parent = rebase(out.joint_parent, b0)
    out.joint_child = rebase(out.joint_child, b0)
    out.joint_ancestor = rebase(out.joint_ancestor, j0)
    out.joint_articulation = rebase(out.joint_articulation, a0)
    out.shape_body = rebase(out.shape_body, b0)
    out.joint_q_start = model.joint_q_start[j0 : j1 + 1].clone() - c0
    out.joint_qd_start = model.joint_qd_start[j0 : j1 + 1].clone() - d0
    out.joint_target_q_start = out.joint_q_start
    out.articulation_start = model.articulation_start[a0 : a1 + 1].clone() - j0
    out.articulation_start[-1] = j1 - j0
    out.articulation_end = model.articulation_end[a0:a1].clone() - j0
    out.articulation_world = rebase(model.articulation_world[a0:a1].clone(), w0)

    def starts(ws, lo, tail):
        v = ws[w0 : w1 + 1].astype(np.int64) - lo
        return torch.tensor([*v.tolist(), int(v[-1]) + tail], dtype=torch.int32, device=model.device)

    out.body_world_start = starts(bws, b0, 0)
    out.joint_world_start = starts(jws, j0, 0)
    out.shape_world_start = starts(sws, s0, g1 - g0)
    out.articulation_world_start = starts(aws, a0, 0)
    out.joint_dof_world_start = starts(dws, d0, 0)
    out.joint_coord_world_start = starts(cws, c0, 0)

    pairs = model.numpy("shape_contact_pairs").astype(np.int64)
    sw = model.numpy("shape_world")
    wa, wb = sw[pairs[:, 0]], sw[pairs[:, 1]]
    pw = np.where(wa >= 0, wa, wb)
    keep = ((pw >= w0) & (pw < w1)) | ((wa == -1) & (wb == -1))
    p = pairs[keep]
    remap = np.where(p >= g0, p - g0 + n_local_shapes, p - s0)
    out.shape_contact_pairs = torch.from_numpy(remap.astype(np.int32)).to(model.device)
    out.shape_contact_pair_count = int(remap.shape[0])
    out.gravity = torch.cat([model.gravity[w0:w1], model.gravity[-1:]]).clone()
    out.actuators = []
    for act in getattr(model, "actuators", []):  # the actuators of this slice's dofs, rebased; groups left empty are dropped
        dof = act.indices.cpu().numpy()
        keep = (dof >= d0) & (dof < d1)
        if keep.any():
            out.actuators.append(act._rebuilt(model.device, keep, d0, c0))
    if getattr(model, "bvh_shape_enabled", None) is not None:  # ray-casting tables for this slice, with the model's mask
        out.bvh_build_shapes(out, shape_flags=model._bvh_build_flags)
    return out


class PeerStateGather:
    """End-of-frame all-gather of per-rank state slices through NVLink peer WRITES on the copy engines (``nb2_peer_gather_*`` in
    ``csrc/nb2_peer.cu``) instead of NCCL all-gather kernels, which would take SMs from a solver kernel that needs all of them to
    stay one wave (DESIGN.md §6).  One process per GPU of one node; ``torch.distributed`` (any backend) is used once, at
    construction, to exchange the CUDA IPC handles.

    ``templates`` are this rank's tensors (e.g. ``state.body_q``, ``state.body_qd``); every rank must pass the same shapes.
    ``push(tensors)`` snapshots them (device-to-device, on the current stream), then - on a side stream - writes the snapshot into
    every rank's receive slot and publishes the sequence number; ``wait(seq)`` makes the current stream wait until all ranks'
    slices of that push have arrived; ``gathered(seq)`` returns ``[world_size, *shape]`` views of the receive slot."""

    def __init__(self, templates, group=None):
        import ctypes as C

        import torch.distributed as dist

        from .. import _lib

        self._C, self._lib = C, _lib.lib()
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.device = templates[0].device
        self.shapes = [tuple(t.shape) for t in templates]
        self.dtypes = [t.dtype for t in templates]
        self.offsets, off = [], 0
        for t in templates:
            self.offsets.append(off)
            off += (t.numel() * t.element_size() + 15) & ~15
        self.bytes = off
        # Every rank reaches every collective below whether or not its own local step failed (a rank that raised early would leave
        # the others waiting inside all_gather_object for the NCCL timeout): local failures are recorded, agreed on, raised together.
        h = C.c_void_p()
        self._h = None
        nh = int(self._lib.nb2_peer_gather_handle_bytes())
        mine = C.create_string_buffer(nh)
        err = None
        try:
            _lib.check(self._lib.nb2_peer_gather_create(self.device.index, self.rank, self.world, self.bytes, C.byref(h)),
                       "nb2_peer_gather_create")
            self._h = h
            _lib.check(self._lib.nb2_peer_gather_export(h, mine), "nb2_peer_gather_export")
        except Exception as e:  # noqa: BLE001 - reported below, on every rank
            err = f"rank {self.rank}: {e}"
        handles = [None] * self.world
        dist.all_gather_object(handles, (err, bytes(mine.raw)), group=group)
        errors = [e for e, _ in handles if e]
        if not errors:
            try:
                _lib.check(self._lib.nb2_peer_gather_connect(h, C.c_char_p(b"".join(b for _, b in handles))), "nb2_peer_gather_connect")
            except Exception as e:  # noqa: BLE001
                err = f"rank {self.rank}: {e}"
            connected = [None] * self.world
            dist.all_gather_object(connected, err, group=group)  # doubles as the barrier: every rank has mapped every buffer
            errors = [e for e in connected if e]
        if errors:
            self.close()
            raise RuntimeError("peer gather unavailable: " + "; ".join(errors))
        self.stride = int(self._lib.nb2_peer_gather_stride(h))
        self._snap = torch.empty(self.stride, dtype=torch.uint8, device=self.device)
        self._copy_stream = torch.cuda.Stream(device=self.device)
        self._snap_free = None  # event: the previous push has finished reading the snapshot
        self.sequence = 0

    def _slot_view(self, slot: int):
        """The receive slot as a flat uint8 tensor (zero-copy view of the library's cudaMalloc block)."""
        ptr = int(self._lib.nb2_peer_gather_buffer(self._h, slot))
        n = self.world * self.stride

        class _Raw:
            __cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3, "strides": None}

        return torch.as_tensor(_Raw(), device=self.device)

    def push(self, tensors) -> int:
        cur = torch.cuda.current_stream(self.device)
        if self._snap_free is not None:
            cur.wait_event(self._snap_free)
        for t, off in zip(tensors, self.offsets):
            n = t.numel() * t.element_size()
            self._snap[off : off + n].copy_(t.contiguous().view(torch.uint8).view(-1), non_blocking=True)
        ready = torch.cuda.Event()
        ready.record(cur)
        self.sequence += 1
        with torch.cuda.stream(self._copy_stream):
            self._copy_stream.wait_event(ready)
            self._lib_check(self._lib.nb2_peer_gather_push(self._h, self._C.c_void_p(self._snap.data_ptr()), self.bytes, self.sequence,
                                                           self._C.c_void_p(self._copy_stream.cuda_stream)), "nb2_peer_gather_push")
            self._snap_free = torch.cuda.Event()
            self._snap_free.record(self._copy_stream)
        return self.sequence

    def _lib_check(self, st, what):
        from .. import _lib

        _lib.check(st, what)

    def wait(self, sequence: int | None = None) -> None:
        seq = self.sequence if sequence is None else int(sequence)
        if seq <= 0:
            return
        cur = torch.cuda.current_stream(self.device)
        self._lib_check(self._lib.nb2_peer_gather_wait(self._h, seq, self._C.c_void_p(cur.cuda_stream)), "nb2_peer_gather_wait")

    def gathered(self, sequence: int | None = None):
        seq = self.sequence if sequence is None else int(sequence)
        raw = self._slot_view(seq & 1).view(self.world, self.stride)
        out = []
        for shape, dtype, off in zip(self.shapes, self.dtypes, self.offsets):
            n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
            out.append(raw[:, off : off + n].view(dtype).view(self.world, *shape))
        return out

    def close(self):
        if getattr(self, "_h", None):
            torch.cuda.synchronize(self.device)
            self._lib.nb2_peer_gather_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
