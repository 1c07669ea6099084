"""PhysicsWorld / PhysicsPipeline: the reference-facing call surface over the C ABI.

Mirrors PhysicsWorld::{new, insert, step} (src/pipeline/physics_world.rs:120-207) and
PhysicsPipeline::step (src/pipeline/physics_pipeline/mod.rs:196-247).  Every method is a thin
ctypes call into librapier_b200.so; no physics is computed in Python.
"""
import ctypes as C

import numpy as np

from . import _abi as A
from ._lib import lib as _product_lib
from .sets import ColliderSet, ImpulseJointSet, RigidBodySet, as_array


class RapierError(RuntimeError):
    pass


class PhysicsPipeline:
    """Owns the device-resident world (the reference's pipeline owns only scratch memory,
    physics_pipeline/mod.rs:34-44; here the scratch IS the HBM mirror of the caller's sets)."""

    def __init__(self, integration_parameters=None, device=0, _lib=None):
        self.L = _lib or _product_lib()
        self.params = integration_parameters or A.RbIntegrationParameters.default()
        self.h = self.L.rb_world_create(C.byref(self.params), device)
        if not self.h:
            raise RapierError(self.L.rb_last_error().decode())
        self.nb = 0
        self._nhulls = 0
        self.hull_vertices = []                # vertices [n, 3] of each registered hull (id = index + 1)
        self.user_force = np.zeros((0, 3))     # the user force of every body as last set (sharding.py bounds accelerations with it)
        self.gravity = None                    # the gravity of the last step (PhysicsWorld sets it at construction)

    def sync_hulls(self, colliders):
        """Registers the convex polyhedra the collider set has collected since the last call (rb_world_add_hull)."""
        from .sets import hull_arrays
        for k in range(self._nhulls, len(getattr(colliders, "hulls", []))):
            verts, sizes, idx = hull_arrays(colliders.hulls[k])
            hid = self._check(self.L.rb_world_add_hull(self.h, len(verts), verts.ctypes.data, len(sizes), sizes.ctypes.data, idx.ctypes.data))
            assert hid == k + 1, (hid, k)
            self.hull_vertices.append(verts.copy())
            self._nhulls = k + 1

    def close(self):
        if getattr(self, "h", None):
            self.L.rb_world_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc < 0:
            raise RapierError(f"rapier_b200 status {rc}: {self.L.rb_last_error().decode()}")
        return rc

    def upload(self, bodies: RigidBodySet, colliders: ColliderSet, joints: ImpulseJointSet = None):
        """handle_user_changes_to_{colliders,rigid_bodies} (substep.rs:303-334): full scene upload."""
        joints = joints or ImpulseJointSet()
        self.sync_hulls(colliders)
        self._b = as_array(bodies.descs, A.RbBodyDesc)
        self._c = as_array(colliders.descs, A.RbColliderDesc)
        self._j = as_array(joints.descs, A.RbJointDesc)
        self._check(self.L.rb_world_set_scene(self.h, len(bodies), self._b, len(colliders), self._c, len(joints), self._j))
        self.nb = len(bodies)
        self.user_force = np.array([d.user_force[:] for d in bodies.descs], np.float64).reshape(-1, 3)

    def reserve(self, max_bodies, max_colliders):
        """Room for later insert() calls (applied by the next upload)."""
        self._check(self.L.rb_world_reserve(self.h, max_bodies, max_colliders))

    def insert(self, body_descs, collider_descs):
        """handle_user_changes_to_{rigid_bodies,colliders} for INSERTED bodies / colliders (user_changes.rs:11-46):
        appended without disturbing any contact state.  Returns (first body index, first collider index)."""
        b = as_array(body_descs, A.RbBodyDesc)
        c = as_array(collider_descs, A.RbColliderDesc)
        fb, fc = C.c_int32(-1), C.c_int32(-1)
        self._check(self.L.rb_world_insert(self.h, len(body_descs), b, len(collider_descs), c, C.byref(fb), C.byref(fc)))
        self.nb += len(body_descs)
        self.user_force = np.concatenate([self.user_force, np.array([d.user_force[:] for d in body_descs], np.float64).reshape(-1, 3)])
        return fb.value, fc.value

    def remove_bodies(self, indices):
        idx = np.ascontiguousarray(indices, np.int32)
        self._check(self.L.rb_world_remove_bodies(self.h, len(idx), idx.ctypes.data))

    def reserve_joints(self, max_joints, generic=False):
        """Room for later insert_joints() calls (applied by the next upload); generic: also the limits / motors / coupled-axes path."""
        self._check(self.L.rb_world_reserve_joints(self.h, max_joints, 1 if generic else 0))

    def insert_joints(self, joint_descs):
        """ImpulseJointSet::insert after the upload: appended, every existing index kept.  Returns the first new index."""
        j = as_array(joint_descs, A.RbJointDesc)
        first = C.c_int32(-1)
        self._check(self.L.rb_world_insert_joints(self.h, len(joint_descs), j, C.byref(first)))
        return first.value

    def remove_joints(self, indices):
        idx = np.ascontiguousarray(indices, np.int32)
        self._check(self.L.rb_world_remove_joints(self.h, len(idx), idx.ctypes.data))

    def update_joints(self, indices, joint_descs, wake_up=True):
        """ImpulseJointSet::get_mut(handle, wake_up) + edits: new descriptors in place (same bodies), impulses kept."""
        idx = np.ascontiguousarray(indices, np.int32)
        j = as_array(joint_descs, A.RbJointDesc)
        self._check(self.L.rb_world_update_joints(self.h, len(idx), idx.ctypes.data, j, 1 if wake_up else 0))

    def set_collider_filters(self, indices, filters):
        """Collider::set_collision_groups / set_solver_groups / set_active_collision_types: collider indices[k] takes filters[k]
        (RbColliderFilter) from the next step on."""
        idx = np.ascontiguousarray(indices, np.int32)
        f = as_array(filters, A.RbColliderFilter)
        self._check(self.L.rb_world_set_collider_filters(self.h, len(idx), idx.ctypes.data, f))

    def set_params(self, params):
        self.params = params
        self._check(self.L.rb_world_set_params(self.h, C.byref(params)))

    def step(self, gravity, nsteps=1, sync=True):
        self.gravity = tuple(gravity)
        g = (C.c_float * 3)(*gravity)
        self._check(self.L.rb_world_step(self.h, g, nsteps, 1 if sync else 0))

    def step_host(self, gravity, in_state13=None, out_state13=None):
        """PhysicsPipeline::step as a host-side owner of the sets calls it: host state in, host state out."""
        self.gravity = tuple(gravity)
        g = (C.c_float * 3)(*gravity)
        self._check(self.L.rb_world_step_host(self.h, g,
                                              None if in_state13 is None else in_state13.ctypes.data,
                                              None if out_state13 is None else out_state13.ctypes.data))

    def set_stream(self, cuda_stream):
        self._check(self.L.rb_world_set_stream(self.h, cuda_stream))

    def import_states(self, idx_dev_ptr, src_dev_ptr, n):
        self._check(self.L.rb_world_import_states(self.h, idx_dev_ptr, src_dev_ptr, n))

    def synchronize(self):
        self._check(self.L.rb_world_synchronize(self.h))

    def body_states(self):
        pose = np.zeros((self.nb, 7), np.float32)
        vel = np.zeros((self.nb, 6), np.float32)
        self._check(self.L.rb_world_get_body_states(self.h, pose.ctypes.data, vel.ctypes.data))
        return pose, vel

    def set_body_states(self, indices, pose7=None, vel6=None):
        idx = np.ascontiguousarray(indices, np.int32)
        p = None if pose7 is None else np.ascontiguousarray(pose7, np.float32)
        v = None if vel6 is None else np.ascontiguousarray(vel6, np.float32)
        self._check(self.L.rb_world_set_body_states(self.h, len(idx), idx.ctypes.data,
                                                    None if p is None else p.ctypes.data,
                                                    None if v is None else v.ctypes.data))

    def set_body_forces(self, indices, force3=None, torque3=None):
        """RigidBody::reset_forces + add_force / add_torque: replaces the user force / torque of the listed bodies."""
        idx = np.ascontiguousarray(indices, np.int32)
        f = None if force3 is None else np.ascontiguousarray(force3, np.float32)
        t = None if torque3 is None else np.ascontiguousarray(torque3, np.float32)
        self._check(self.L.rb_world_set_body_forces(self.h, len(idx), idx.ctypes.data, None if f is None else f.ctypes.data,
                                                    None if t is None else t.ctypes.data))
        if f is not None:
            self.user_force[idx] = f.reshape(-1, 3)

    def set_next_kinematic_positions(self, indices, pose7):
        """RigidBody::set_next_kinematic_position of position-based kinematic bodies ([n, 7]: translation, quaternion xyzw)."""
        idx = np.ascontiguousarray(indices, np.int32)
        p = np.ascontiguousarray(pose7, np.float32)
        self._check(self.L.rb_world_set_next_kinematic_positions(self.h, len(idx), idx.ctypes.data, p.ctypes.data))

    def collision_events(self, with_flags=False):
        """Drains the buffered CollisionEvents (EventHandler::handle_collision_event): [(collider1, collider2, started, step)],
        with_flags: [(..., flags)] (RB_COLLISION_EVENT_SENSOR)."""
        buf = (A.RbCollisionEvent * 65536)()
        n = self.L.rb_world_drain_collision_events(self.h, 65536, buf)
        self._check(min(n, 0))
        if with_flags:
            return [(e.collider1, e.collider2, e.started, e.step, e.flags) for e in buf[:min(n, 65536)]]
        return [(e.collider1, e.collider2, e.started, e.step) for e in buf[:min(n, 65536)]]

    def contact_force_events(self):
        """Drains the buffered ContactForceEvents (EventHandler::handle_contact_force_event)."""
        buf = (A.RbContactForceEvent * 65536)()
        n = self.L.rb_world_drain_contact_force_events(self.h, 65536, buf)
        self._check(min(n, 0))
        return [dict(collider1=e.collider1, collider2=e.collider2, total_force=tuple(e.total_force), total_force_magnitude=e.total_force_magnitude,
                     max_force_direction=tuple(e.max_force_direction), max_force_magnitude=e.max_force_magnitude, started=e.started, step=e.step)
                for e in buf[:min(n, 65536)]]

    def counters(self):
        c = A.RbCounters()
        self._check(self.L.rb_world_get_counters(self.h, C.byref(c)))
        return c.as_dict()

    def enable_profiling(self, flag=True):
        self._check(self.L.rb_world_enable_profiling(self.h, 1 if flag else 0))

    def contact_pairs(self):
        n = self._check(self.L.rb_world_get_contact_pairs(self.h, 0, None, None, None, None, None))
        pc = np.zeros((n, 2), np.int32)
        nc = np.zeros(n, np.int32)
        col = np.zeros(n, np.int32)
        nrm = np.zeros((n, 3), np.float32)
        imp = np.zeros((n, 4), np.float32)
        if n:
            self._check(self.L.rb_world_get_contact_pairs(self.h, n, pc.ctypes.data, nc.ctypes.data, col.ctypes.data,
                                                          nrm.ctypes.data, imp.ctypes.data))
        return dict(colliders=pc, num_contacts=nc, color=col, normal=nrm, impulses=imp)

    def debug_read(self, table, dtype):
        n = self.L.rb_world_debug_read(self.h, table.encode(), None, 0)
        if n < 0:
            raise KeyError(f"{table}: {self.L.rb_last_error().decode()}")
        buf = np.zeros(max(int(n), 1), np.uint8)
        self.L.rb_world_debug_read(self.h, table.encode(), buf.ctypes.data, n)
        return buf[:n].view(dtype)

    def label_components(self):
        out = np.zeros(self.nb, np.int32)
        self._check(self.L.rb_world_label_components(self.h, out.ctypes.data))
        return out

    def set_owned_bodies(self, owned):
        o = np.ascontiguousarray(owned, np.uint8)
        assert o.shape == (self.nb,)
        self._check(self.L.rb_world_set_owned_bodies(self.h, o.ctypes.data))

    def quarantine(self):
        """PhysicsPipeline::quarantine().bodies(): bodies disabled since the last call because their state went non-finite."""
        n = self._check(self.L.rb_world_get_quarantine(self.h, None, 0))
        out = np.zeros(max(n, 1), np.int32)
        if n:
            self._check(self.L.rb_world_get_quarantine(self.h, out.ctypes.data, n))
        return out[:n]

    def sleeping(self):
        """RigidBody::is_sleeping of every body."""
        out = np.zeros(self.nb, np.uint8)
        self._check(self.L.rb_world_get_sleeping(self.h, out.ctypes.data))
        return out

    def wake_up(self, indices):
        """IslandManager::wake_up(handle, strong = true): wakes the bodies' whole islands."""
        idx = np.ascontiguousarray(indices, np.int32)
        self._check(self.L.rb_world_wake_up(self.h, len(idx), idx.ctypes.data))

    def set_halo_bodies(self, flags_dev_ptr):
        """Which bodies of other ranks are tracked here (device array of num_bodies bytes; see sharding.py)."""
        self._check(self.L.rb_world_set_halo_bodies(self.h, flags_dev_ptr))

    def import_halo(self):
        self._check(self.L.rb_world_import_halo(self.h))

    def state_buffer(self):
        p = C.c_void_p()
        n = C.c_int64()
        self._check(self.L.rb_world_state_buffer(self.h, C.byref(p), C.byref(n)))
        return p.value, n.value

    def state_buffers(self):
        """Turns on double buffering of the packed state (see include/rapier_b200.h); returns (ptr0, ptr1, bytes)."""
        p0, p1, n = C.c_void_p(), C.c_void_p(), C.c_int64()
        self._check(self.L.rb_world_state_buffers(self.h, C.byref(p0), C.byref(p1), C.byref(n)))
        return p0.value, p1.value, n.value

    def import_states_from(self, idx_dev_ptr, table_dev_ptr, n):
        self._check(self.L.rb_world_import_states_from(self.h, idx_dev_ptr, table_dev_ptr, n))


class PhysicsWorld:
    """PhysicsWorld facade (src/pipeline/physics_world.rs): sets + pipeline + gravity."""

    def __init__(self, scene=None, integration_parameters=None, device=0, _lib=None):
        self.gravity = (0.0, -9.81, 0.0)
        self.bodies = RigidBodySet()
        self.colliders = ColliderSet()
        self.impulse_joints = ImpulseJointSet()
        self.integration_parameters = integration_parameters or A.RbIntegrationParameters.default()
        self.physics_pipeline = PhysicsPipeline(self.integration_parameters, device, _lib=_lib)
        self._dirty = True
        self._uploaded = (0, 0, 0)   # bodies, colliders, joints the device already has
        if scene is not None:
            self.gravity = scene.gravity
            self.bodies, self.colliders, self.impulse_joints = scene.bodies, scene.colliders, scene.joints
        self.physics_pipeline.gravity = tuple(self.gravity)

    def reserve(self, max_bodies, max_colliders):
        """Capacity for bodies / colliders inserted after the first step (RigidBodySet / ColliderSet grow on demand in the
        reference; the device tables are sized once)."""
        self.physics_pipeline.reserve(max_bodies, max_colliders)

    def insert(self, body_builder, collider_builder):
        """PhysicsWorld::insert (physics_world.rs:184-207).  After the world has been stepped, the new body and collider
        are appended on the device (contacts, warm-start data and islands of everything else persist)."""
        h = self.bodies.insert(body_builder)
        self.colliders.insert_with_parent(collider_builder, h)
        self._dirty = True
        return h

    def insert_collider(self, collider_builder, parent=None):
        """PhysicsWorld::insert_collider (parentless = static geometry)."""
        self._dirty = True
        return self.colliders.insert(collider_builder) if parent is None else self.colliders.insert_with_parent(collider_builder, parent)

    def remove(self, body_handle):
        """RigidBodySet::remove with its attached colliders; the handle's slot stays allocated."""
        self._flush()
        self.physics_pipeline.remove_bodies([body_handle])

    def insert_impulse_joint(self, body1, body2, joint_builder):
        """ImpulseJointSet::insert.  After the first step the joint is appended on the device (rb_world_insert_joints; capacity
        from reserve_joints) without touching any other state."""
        h = self.impulse_joints.insert(body1, body2, joint_builder)
        nb0, nc0, nj0 = self._uploaded
        if nb0 + nc0 > 0 and not self._dirty:
            self.physics_pipeline.insert_joints(self.impulse_joints.descs[nj0:])
            self._uploaded = (nb0, nc0, len(self.impulse_joints))
        else:
            self._dirty = True
        return h

    def remove_impulse_joint(self, joint_handle):
        """ImpulseJointSet::remove (the handle's slot stays allocated)."""
        self._flush()
        self.physics_pipeline.remove_joints([joint_handle])

    def reserve_joints(self, max_joints, generic=False):
        self.physics_pipeline.reserve_joints(max_joints, generic)

    def _flush(self):
        if self._dirty:
            nb0, nc0, nj0 = self._uploaded
            nb, nc, nj = len(self.bodies), len(self.colliders), len(self.impulse_joints)
            if nb0 + nc0 > 0 and nj == nj0 and nb >= nb0 and nc >= nc0:   # only appended since the last upload: incremental
                self.physics_pipeline.sync_hulls(self.colliders)
                self.physics_pipeline.insert(self.bodies.descs[nb0:], self.colliders.descs[nc0:])
            else:
                self.physics_pipeline.upload(self.bodies, self.colliders, self.impulse_joints)
                nc0 = 0
            # the colliders just uploaded whose filters are not the defaults (a scene without any makes no such call)
            new = sorted(i for i in self.colliders.filters if i >= nc0)
            if new:
                self.physics_pipeline.set_collider_filters(new, [self.colliders.filters[i] for i in new])
            self._uploaded = (nb, nc, nj)
            self._dirty = False

    def step(self, n=1, sync=True):
        self._flush()
        self.physics_pipeline.step(self.gravity, n, sync)

    def body_states(self):
        self._flush()
        return self.physics_pipeline.body_states()

    def counters(self):
        self._flush()
        return self.physics_pipeline.counters()

    def quarantine(self):
        self._flush()
        return self.physics_pipeline.quarantine()

    def sleeping(self):
        self._flush()
        return self.physics_pipeline.sleeping()

    def wake_up(self, handles):
        self._flush()
        self.physics_pipeline.wake_up(handles)

    def contact_pairs(self):
        self._flush()
        return self.physics_pipeline.contact_pairs()

    def set_body_states(self, handles, pose7=None, vel6=None):
        """RigidBody::set_position / set_linvel / set_angvel (wakes the bodies' islands)."""
        self._flush()
        self.physics_pipeline.set_body_states(handles, pose7, vel6)

    def set_collider_filters(self, handles, collision_groups=None, solver_groups=None, active_collision_types=None):
        """Collider::set_collision_groups / set_solver_groups / set_active_collision_types on the listed colliders, effective
        from the next step.  collision_groups and solver_groups are (memberships, filter) or (memberships, filter, test_mode);
        an argument left at None keeps the collider's current value."""
        self._flush()
        handles = [int(h) for h in handles]
        new = []
        for h in handles:
            f = self.colliders.filter(h)
            if collision_groups is not None:
                g = tuple(collision_groups) + (A.RB_TEST_AND,) * (3 - len(collision_groups))
                f.collision_memberships, f.collision_filter, f.collision_test_mode = g
            if solver_groups is not None:
                g = tuple(solver_groups) + (A.RB_TEST_AND,) * (3 - len(solver_groups))
                f.solver_memberships, f.solver_filter, f.solver_test_mode = g
            if active_collision_types is not None:
                f.active_collision_types = int(active_collision_types)
            new.append(f)
        self.physics_pipeline.set_collider_filters(handles, new)
        for h, f in zip(handles, new):   # (the sets mirror what the device now holds)
            self.colliders.descs[h].collision_memberships = f.collision_memberships
            self.colliders.descs[h].collision_filter = f.collision_filter
            self.colliders.filters[h] = f

    def set_body_forces(self, handles, force3=None, torque3=None):
        self._flush()
        self.physics_pipeline.set_body_forces(handles, force3, torque3)

    def set_next_kinematic_positions(self, handles, pose7):
        self._flush()
        self.physics_pipeline.set_next_kinematic_positions(handles, pose7)

    def collision_events(self, with_flags=False):
        self._flush()
        return self.physics_pipeline.collision_events(with_flags)

    def contact_force_events(self):
        self._flush()
        return self.physics_pipeline.contact_force_events()

    def debug_read(self, table, dtype):
        self._flush()
        return self.physics_pipeline.debug_read(table, dtype)
