"""Island sharding across ranks (SURVEY.md 8e): whole connected components are assigned to ranks and every rank
simulates only the bodies it owns.  What crosses NVLink is the north star's "all-gather of boundary body states":

  * HALO bodies -- bodies of other ranks inside (or near) the bounding box of this rank's bodies -- are tracked here
    for proximity detection only; their states (13 floats: t3 q4 linvel3 angvel3) are all-gathered EVERY step and
    imported before the next one.  A rank with no halo takes part in no per-step collective at all.
  * every `refresh_every` (128) steps the owned states of ALL bodies are all-gathered, every rank re-derives its halo set
    from them (halo_rule: bounding box of its own bodies' reach spheres, inflated per axis by a margin that covers
    `refresh_every` steps at the fastest body's current speed plus the largest acceleration gravity and user forces can
    give) and tells the others which of their bodies it now tracks.  It also checks that no untracked body broke that
    bound over the last window (check_bound), and raises HaloBoundError if one did.
  * a CONTACT between an owned and a halo body means two shards' islands merged: the device raises RB_ERR_SHARD
    (reported by the next synchronising call); nothing is silently simulated wrong.
  * `finish()` gathers everything once more, so all ranks end with the exact state of every body.

The reference is single-process (one awake set, src/dynamics/island_manager/manager.rs:20-25); the components it
tracks as persistent islands (island_manager/persistent.rs:1-3) are the unit of distribution.  Works with any
torch.distributed backend: NCCL over NVLink on the GPU box, gloo in the CPU tests (host emulation of the kernels).
"""
import ctypes as C

import numpy as np
import torch


def partition_components(component_of_body, world_size):
    """Contiguous blocks of components (ascending root id) per rank, balanced by body count.
    Returns owner[b] in [0, world_size) or -1 for non-dynamic bodies."""
    comp = np.asarray(component_of_body)
    roots, counts = np.unique(comp[comp >= 0], return_counts=True)
    cum = np.cumsum(counts) - counts
    total = max(int(counts.sum()), 1)
    owner_of_root = np.minimum((cum * world_size) // total, world_size - 1)
    lut = dict(zip(roots.tolist(), owner_of_root.tolist()))
    return np.array([lut[int(c)] if c >= 0 else -1 for c in comp], np.int32)


class _CudaBuf:
    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {"shape": (nbytes // 4,), "typestr": "<f4", "data": (ptr, False), "version": 2}


def state_tensor(pipe, device):
    """Zero-copy torch view [nb, 13] of the library's packed body-state buffer."""
    ptr, nbytes = pipe.state_buffer()
    if device.type == "cuda":
        t = torch.as_tensor(_CudaBuf(ptr, nbytes), device=device)
    else:
        t = torch.frombuffer((C.c_float * (nbytes // 4)).from_address(ptr), dtype=torch.float32)
    return t.view(-1, 13)


def body_reach(pipe):
    """(local centre of mass [nb, 3], reach [nb]) of every body: the radius about its centre of mass of a sphere that holds
    every one of its colliders' broad-phase boxes (shape extent + the collider's offset from the centre of mass + its
    contact skin + the prediction distance + the fat-box skin).  Centred on the centre of mass, the sphere is carried by
    the body's linear velocity alone: spin turns the colliders inside it."""
    from . import _abi as A
    mp = pipe.debug_read("body_mprops", np.float32).reshape(-1, 16).astype(np.float64)
    com = mp[:, 0:3]
    prm = pipe.params
    pad = (prm.normalized_prediction_distance + A.RB_FAT_SKIN_FACTOR) * prm.length_unit   # prediction distance + fat-box skin
    r = np.zeros(pipe.nb, np.float64)
    for c in pipe._c:
        if c.parent < 0:
            continue
        he = np.array(c.half_extents[:], np.float64)
        if c.shape == A.RB_SHAPE_BALL:
            ext = he[0]
        elif c.shape == A.RB_SHAPE_CUBOID:
            ext = np.linalg.norm(he)
        elif c.shape == A.RB_SHAPE_CAPSULE:      # (half height, radius, axis)
            ext = he[0] + he[1]
        elif c.shape == A.RB_SHAPE_CONVEX:       # (hull id, border radius)
            ext = np.linalg.norm(pipe.hull_vertices[int(he[0]) - 1], axis=1).max() + he[1]
        else:
            raise ValueError(f"body_reach: unknown shape {c.shape}")
        off = np.linalg.norm(np.array(c.pos_wrt_parent_t[:], np.float64) - com[c.parent])
        r[c.parent] = max(r[c.parent], off + ext + c.contact_skin + pad)
    return com.astype(np.float32), r.astype(np.float32)


def rotate(q, v):
    """v rotated by the unit quaternions q = (x, y, z, w), batched."""
    b, w = q[:, 0:3], q[:, 3:4]
    t = 2.0 * torch.cross(b, v, dim=1)
    return v + w * t + torch.cross(b, t, dim=1)


def body_centres(state, com):
    """World centres of mass of the state rows [nb, 13] (translation, quaternion, linvel, angvel)."""
    return state[:, 0:3] + rotate(state[:, 3:7], com)


def owned_box(centre, reach, mine):
    """Bounding box (lo [3], hi [3]) of the reach spheres of the bodies in `mine`, or None when there are none."""
    if not bool(mine.any()):
        return None
    r = reach.unsqueeze(1)
    return (centre - r)[mine].min(dim=0).values, (centre + r)[mine].max(dim=0).values


def halo_margin(state, window, accel, min_margin=0.5):
    """Per-axis margin [3] by which a rank's bounding box is widened: the owned and the foreign body can each cover
    window * v_max + accel * window^2 / 2 before the next refresh, v_max the fastest body's speed now and accel the
    per-axis bound on acceleration (gravity * max|gravity_scale| + max|F| / m)."""
    lin = state[:, 7:10]
    speed = lin.norm(dim=1).max() if lin.numel() else torch.zeros((), device=state.device)
    return min_margin + 2.0 * window * speed + torch.as_tensor(accel, dtype=state.dtype, device=state.device) * window * window


def halo_rule(state, com, reach, owner, rank, window, accel, min_margin=0.5):
    """The foreign bodies rank `rank` must track for the next `window` seconds (uint8 mask [nb]): those whose reach
    sphere meets the bounding box of its own bodies' reach spheres widened by halo_margin.  Before the next refresh no
    untracked foreign body can come within the broad phase's reach of an owned one unless something the margin does not
    bound (a contact impulse, a state edit, a kinematic target) accelerates it; IslandShard checks that at every refresh.
    state [nb, 13], com [nb, 3], reach [nb], owner [nb] (int, -1 for fixed bodies) are tensors on one device."""
    mine = owner == rank
    foreign = (owner >= 0) & ~mine
    centre = body_centres(state, com)
    box = owned_box(centre, reach, mine)
    if box is None:
        return torch.zeros(owner.shape, dtype=torch.uint8, device=owner.device)
    margin = halo_margin(state, window, accel, min_margin)
    r = reach.unsqueeze(1)
    near = ((centre + r >= box[0] - margin).all(dim=1) & (centre - r <= box[1] + margin).all(dim=1))
    return (near & foreign).to(torch.uint8)


def accel_bound(gravity, gravity_scale, user_force, inv_mass):
    """Per-axis bound [3] on the acceleration of the given bodies: |gravity| times their largest |gravity_scale| plus
    their largest |user force| * inverse mass (contact impulses are not bounded: IslandShard.check_bound)."""
    if gravity is None:
        raise ValueError("the halo margin needs the gravity: step the pipeline, build it through PhysicsWorld or pass gravity=")
    g = np.abs(np.asarray(gravity, np.float64)) * float(np.abs(gravity_scale).max(initial=0.0))
    return g + float((np.linalg.norm(user_force, axis=1) * inv_mass).max(initial=0.0))


class HaloBoundError(RuntimeError):
    """A foreign body reached a rank's bodies between two refreshes without being tracked there (see IslandShard)."""


class IslandShard:
    def __init__(self, pipe, dist, rank, world_size, device, refresh_every=128, min_margin=0.5, overlap=None, gravity=None):
        """gravity: the gravity the halo margin assumes; by default the one the pipeline was last stepped with (or given
        by PhysicsWorld at construction), read at every refresh."""
        self.pipe, self.dist, self.rank, self.world_size, self.device = pipe, dist, rank, world_size, device
        self.refresh_every = int(refresh_every)
        self.min_margin = float(min_margin)
        self.gravity = gravity
        self.dt = float(pipe.params.dt)
        self.tick = 0
        comp = pipe.label_components()
        self.owner = partition_components(comp, world_size)
        pipe.set_owned_bodies((self.owner == rank).astype(np.uint8))
        nb = pipe.nb
        self.state = state_tensor(pipe, device)
        owner_t = torch.from_numpy(self.owner.astype(np.int64)).to(device)
        self.mine = owner_t == rank
        self.foreign = (owner_t >= 0) & ~self.mine
        com, reach = body_reach(pipe)
        self.com = torch.from_numpy(com).to(device)
        self.reach = torch.from_numpy(reach).to(device)
        self.moving = np.nonzero(self.owner >= 0)[0]
        self.inv_mass = pipe.debug_read("body_mprops", np.float32).reshape(-1, 16)[self.moving, 3].astype(np.float64)
        self.gravity_scale = np.array([pipe._b[b].gravity_scale for b in self.moving], np.float64)
        idx = [np.nonzero(self.owner == r)[0].astype(np.int64) for r in range(world_size)]
        self.counts = [len(i) for i in idx]
        self.maxc = max(max(self.counts), 1)
        self.my_idx = torch.from_numpy(idx[rank]).to(device)
        # full exchange: packed owned rows of every rank -> rows of the state table
        self.full_send = torch.zeros(self.maxc, 13, device=device)
        self.full_recv = torch.zeros(world_size * self.maxc, 13, device=device)
        others = [r for r in range(world_size) if r != rank]
        self.other_idx = torch.cat([torch.from_numpy(idx[r]) for r in others] or [torch.zeros(0, dtype=torch.int64)]).to(device)
        self.other_rows = torch.cat([torch.arange(self.counts[r]) + r * self.maxc for r in others] or [torch.zeros(0, dtype=torch.int64)]).to(device)
        self.halo = torch.zeros(nb, dtype=torch.uint8, device=device)   # foreign bodies tracked here
        self.masks = torch.zeros(world_size, nb, dtype=torch.uint8, device=device)   # every rank's halo
        self.owner_t = owner_t
        self.export_max = 0          # per-step halo exchange: rows per rank (0 = no per-step collective)
        self.halo_steps = 0          # steps that needed the per-step halo exchange (diagnostic)
        self.refreshes = 0
        self.refresh(classify=True, force=True)

    def accel(self):
        return accel_bound(self.pipe.gravity if self.gravity is None else self.gravity, self.gravity_scale,
                           self.pipe.user_force[self.moving], self.inv_mass)

    # ---- full exchange (every refresh_every steps, at start-up and in finish) ----
    def _gather_all(self):
        n = self.counts[self.rank]
        self.full_send[:n] = self.state.index_select(0, self.my_idx)
        self.dist.all_gather_into_tensor(self.full_recv, self.full_send)
        if len(self.other_idx):
            self.state.index_copy_(0, self.other_idx, self.full_recv.index_select(0, self.other_rows))

    def check_bound(self):
        """After a full exchange: a foreign body that no rank's halo rule made it track over the last window and that now
        lies within min_margin of a rank's owned bounding box on every axis broke the margin's bound (the margin keeps a
        gap of at least min_margin on one axis otherwise).  Raises HaloBoundError naming the body; every rank holds the
        same states and masks, so every rank raises.  A body that tunnelled through and ended apart is not seen."""
        centre = body_centres(self.state, self.com)
        r = self.reach.unsqueeze(1)
        for rk in range(self.world_size):
            mine = self.owner_t == rk
            box = owned_box(centre, self.reach, mine)
            if box is None:
                continue
            untracked = (self.owner_t >= 0) & ~mine & (self.masks[rk] == 0)
            near = (centre + r >= box[0] - self.min_margin).all(dim=1) & (centre - r <= box[1] + self.min_margin).all(dim=1)
            bad = torch.nonzero(near & untracked).flatten()
            if bad.numel():
                b = int(bad[0])
                raise HaloBoundError(f"body {b} (rank {int(self.owner_t[b])}) reached the bodies of rank {rk} between two halo "
                                     f"refreshes without being tracked there (after {self.tick} steps): its contacts may have been missed")

    def refresh(self, classify=True, force=False):
        """All ranks get all states; each checks that no untracked body broke the last window's bound, re-derives the
        bodies of other ranks it has to track (its halo) and, when any rank's halo changed, learns which of its own bodies
        the others track (its exports).  One host synchronisation."""
        self._gather_all()
        if self.refreshes:
            self.check_bound()
        if not classify:
            return
        self.refreshes += 1
        halo = halo_rule(self.state, self.com, self.reach, self.owner_t, self.rank, self.refresh_every * self.dt,
                         self.accel(), self.min_margin)
        changed = (halo != self.halo).any().to(torch.int32).reshape(1)
        self.dist.all_reduce(changed, op=self.dist.ReduceOp.MAX)
        if not force and int(changed.item()) == 0:     # (the host synchronisation of a refresh)
            return
        self.halo = halo
        self.pipe.set_halo_bodies(self.halo.data_ptr())
        self.pipe.import_halo()
        # who tracks whom: all halo masks -> my export list and everybody's (for unpacking)
        masks = torch.zeros(self.world_size, self.halo.numel(), dtype=torch.uint8, device=self.device)
        self.dist.all_gather_into_tensor(masks.view(-1), self.halo)
        self.masks = masks
        tracked = masks.any(dim=0)                      # bodies tracked by a rank other than their owner
        self.export_idx = []
        counts = []
        for rk in range(self.world_size):
            e = torch.nonzero(tracked & (self.owner_t == rk)).flatten()
            self.export_idx.append(e)
            counts.append(int(e.numel()))
        self.export_max = max(counts) if counts else 0
        if self.export_max > 0:
            self.halo_send = torch.zeros(self.export_max, 13, device=self.device)
            self.halo_recv = torch.zeros(self.world_size * self.export_max, 13, device=self.device)
            self.halo_dst = torch.cat([e for rk, e in enumerate(self.export_idx) if rk != self.rank] or [torch.zeros(0, dtype=torch.int64, device=self.device)])
            self.halo_rows = torch.cat([torch.arange(int(e.numel()), device=self.device) + rk * self.export_max
                                        for rk, e in enumerate(self.export_idx) if rk != self.rank] or [torch.zeros(0, dtype=torch.int64, device=self.device)])

    # ---- per step ----
    def exchange(self):
        """Call after every step: boundary (halo) states every step, everything every `refresh_every` steps."""
        self.tick += 1
        if self.tick % self.refresh_every == 0:
            self.refresh(classify=True)
            return
        if self.export_max == 0:
            return
        self.halo_steps += 1
        mine = self.export_idx[self.rank]
        if mine.numel():
            self.halo_send[:mine.numel()] = self.state.index_select(0, mine)
        self.dist.all_gather_into_tensor(self.halo_recv, self.halo_send)
        if self.halo_dst.numel():
            self.state.index_copy_(0, self.halo_dst, self.halo_recv.index_select(0, self.halo_rows))
        self.pipe.import_halo()

    def finish(self):
        """Afterwards every rank holds the current state of every body."""
        self.refresh(classify=False)
