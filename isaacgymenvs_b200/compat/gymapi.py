"""`isaacgym.gymapi` look-alike backed by the CUDA engine (SURVEY.md 8b "required exports").

Only what `tasks/base/vec_task.py`, the single-actor-per-env tasks and ShadowHand's three-actor envs (articulation +
free box + gravity-less marker, `shadow_hand.py:338-383`) touch is provided; every method cites a representative call site.  Actors, assets and envs are RECORDED
here (create_actor is called num_envs times in a Python loop, `ant.py:185-197`, so it must cost
microseconds); the engine is created once, in `prepare_sim`.
"""
import copy
import os
import types

import numpy as np
import torch

from .. import engine
from ..assets import load_asset_file
from ..importer.model import BuildOptions

SIM_PHYSX, SIM_FLEX = 0, 1
UP_AXIS_Y, UP_AXIS_Z = 0, 1
DOF_MODE_NONE, DOF_MODE_POS, DOF_MODE_VEL, DOF_MODE_EFFORT = 0, 1, 2, 3
DOMAIN_ENV, DOMAIN_SIM, DOMAIN_ACTOR = 0, 1, 2
MESH_VISUAL, MESH_COLLISION, MESH_VISUAL_AND_COLLISION = 0, 1, 2
ENV_SPACE, LOCAL_SPACE, GLOBAL_SPACE = 0, 1, 2
CC_NEVER, CC_LAST_SUBSTEP, CC_ALL_SUBSTEPS = 0, 1, 2


def ContactCollection(v):
    return int(v)


class Vec3:
    __slots__ = ("x", "y", "z")

    def __init__(self, x=0.0, y=0.0, z=0.0):
        self.x, self.y, self.z = float(x), float(y), float(z)

    def __add__(self, o):
        return Vec3(self.x + o.x, self.y + o.y, self.z + o.z)

    def __sub__(self, o):
        return Vec3(self.x - o.x, self.y - o.y, self.z - o.z)

    def __iter__(self):
        return iter((self.x, self.y, self.z))

    def __repr__(self):
        return f"Vec3({self.x}, {self.y}, {self.z})"


class Quat:
    __slots__ = ("x", "y", "z", "w")

    def __init__(self, x=0.0, y=0.0, z=0.0, w=1.0):
        self.x, self.y, self.z, self.w = float(x), float(y), float(z), float(w)


class Transform:
    def __init__(self, p=None, r=None):
        self.p = p if p is not None else Vec3()
        self.r = r if r is not None else Quat()


class _Bag:
    """Attribute bag: unknown keys are accepted, as `setattr(sim_params.physx, opt, ...)` relies on
    (vec_task.py:532-554)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


class PlaneParams(_Bag):
    def __init__(self):
        super().__init__(normal=Vec3(0, 0, 1), distance=0.0, static_friction=1.0, dynamic_friction=1.0, restitution=0.0)


class TriangleMeshParams(_Bag):
    def __init__(self):
        super().__init__(nb_vertices=0, nb_triangles=0, transform=Transform(), static_friction=1.0, dynamic_friction=1.0,
                         restitution=0.0)


class AssetOptions(_Bag):
    def __init__(self):
        super().__init__(fix_base_link=False, default_dof_drive_mode=DOF_MODE_NONE, angular_damping=0.5, linear_damping=0.0,
                         max_angular_velocity=64.0, collapse_fixed_joints=False, replace_cylinder_with_capsule=False,
                         flip_visual_attachments=False, density=1000.0, armature=0.0, thickness=0.02, disable_gravity=False,
                         use_physx_armature=True)


class SimParams(_Bag):
    def __init__(self):
        super().__init__(dt=1.0 / 60.0, substeps=2, up_axis=UP_AXIS_Y, gravity=Vec3(0.0, -9.81, 0.0), use_gpu_pipeline=False,
                         num_client_threads=0, physx=_Bag(num_threads=0, solver_type=1, use_gpu=False), flex=_Bag())


class CameraProperties(_Bag):
    pass


class _Asset:
    def __init__(self, model, options):
        self.model = model
        self.options = options
        self.sensors = []           # (body index, Transform)
        # fixed tendons as gym.get_asset_tendon_properties sees them (shadow_hand.py:255-266): inactive until a
        # limit stiffness is set
        self.tendon_props = [types.SimpleNamespace(limit_stiffness=0.0, damping=0.0, stiffness=0.0, lower_limit=float(t["range"][0]),
                                                   upper_limit=float(t["range"][1])) for t in (model.tendons or [])]
        self.shape_props = [types.SimpleNamespace(friction=float(f), restitution=0.0) for f in model.geom_friction]


class _Env:
    def __init__(self, index):
        self.index = index
        self.actors = []
        self.actor_ids = []


class _Sim:
    def __init__(self, compute_device, params):
        self.compute_device = compute_device
        self.params = params
        self.ground = None
        self.terrain = None         # height field behind an add_triangle_mesh
        self.envs = []
        self.asset = None           # the articulation (actor 0 of every env)
        self.extra_assets = []      # further actors of an env, in creation order: single rigid bodies
        self.start_poses = []       # per env: [Transform per actor]
        self.engine = None
        self.num_actors = 0
        self.frame = 0
        self.obj_force = None       # engine tensor behind apply_rigid_body_force_tensors (the free object's row), once used
        self.obj_force_set = False


class _Tensor:
    """What acquire_*_tensor returns; gymtorch.wrap_tensor unwraps it to the torch tensor."""

    def __init__(self, t):
        self.tensor = t


class Gym:
    # ---- lifecycle (vec_task.py:63,247,262,382,386)
    def create_sim(self, compute_device, graphics_device, sim_type, params):
        return _Sim(compute_device, params)

    def add_ground(self, sim, plane_params):
        sim.ground = plane_params

    def add_triangle_mesh(self, sim, vertices, triangles, params):
        """anymal_terrain.py:196-208.  The engine collides with height fields, not general meshes.  A mesh that comes from
        `terrain_utils.convert_heightfield_to_trimesh` carries the samples it was built from (its arrays are tagged) and the
        engine gets that height field itself; any other mesh is taken as a terrain surface z(x, y) and sampled onto a grid
        (`terrain.trimesh_to_heightfield`: node spacing from the mesh's edge lengths; overhangs collapse to their upper surface).
        Either way the field is placed at params.transform.p."""
        src = getattr(vertices, "source", None)
        ox, oy = float(params.transform.p.x), float(params.transform.p.y)
        if src is None:
            from ..terrain import trimesh_to_heightfield
            nv, nt = int(getattr(params, "nb_vertices", 0) or 0), int(getattr(params, "nb_triangles", 0) or 0)
            v = np.asarray(vertices, dtype=np.float64).reshape(-1, 3); t = np.asarray(triangles).reshape(-1, 3)
            if (nv and nv != len(v)) or (nt and nt != len(t)):
                raise ValueError("add_triangle_mesh: nb_vertices / nb_triangles do not match the arrays")
            src = trimesh_to_heightfield(v, t)
            ox, oy = ox + src["offset"][0], oy + src["offset"][1]
            src = {k: src[k] for k in ("height_field", "horizontal_scale", "vertical_scale")}
        sim.terrain = dict(src, origin=(ox, oy), z0=float(params.transform.p.z), friction=float(params.dynamic_friction))

    def prepare_sim(self, sim):
        if sim.engine is not None:
            return True
        if sim.asset is None or not sim.envs:
            raise RuntimeError("prepare_sim: no actors were created")
        a, p = sim.asset, sim.params
        model = copy.deepcopy(a.model)
        model.sensor_body = np.array([b for b, _ in a.sensors], dtype=np.int32)
        model.sensor_pos = np.zeros((len(a.sensors), 3)); model.sensor_quat = np.tile([0, 0, 0, 1.0], (len(a.sensors), 1))
        mu = sim.ground.dynamic_friction if sim.ground is not None else 1.0
        g = p.gravity
        hf_kw = {}
        if sim.terrain is not None:
            t = sim.terrain
            if t["z0"] != 0.0:
                raise NotImplementedError("add_triangle_mesh: vertical offset of the terrain")
            mu = t["friction"]
            hf_kw = dict(hfield=t["height_field"], hf_horizontal_scale=t["horizontal_scale"], hf_vertical_scale=t["vertical_scale"],
                         hf_origin=t["origin"])
        ext = None
        apr = 1 + len(sim.extra_assets)
        if sim.extra_assets:
            # further actors: single free bodies.  The first one with gravity is the simulated object (a box);
            # gravity-less ones are markers the engine never moves (goal object, shadow_hand.py:281-282,380)
            obj, obj_row = None, -1
            for k, xa in enumerate(sim.extra_assets):
                xm = xa.model
                if xm.ndof != 0 or xm.nb != 1:
                    raise NotImplementedError("extra actors of an env must be single rigid bodies")
                if xa.options.disable_gravity:
                    continue
                if obj is not None or k != 0:
                    raise NotImplementedError("one simulated free object per env, created right after the articulation")
                from ..tasks.shadow_hand import object_shape      # box / capsule / sphere / prolate spheroid -> rounded box
                half, rnd = object_shape(xm)
                obj = dict(mass=float(xm.mass[0]), inertia=[float(xm.inertia[0][c]) for c in range(3)],
                           half=half, round=rnd, mu=float(xa.shape_props[0].friction), gravity_on=1,
                           angular_damping=float(xa.options.angular_damping), linear_damping=float(xa.options.linear_damping),
                           max_angular_velocity=float(xa.options.max_angular_velocity))
                obj_row = 1
            tend = [dict(t) for t, tp in zip(model.tendons or [], a.tendon_props) if tp.limit_stiffness > 0.0]
            ks = {(tp.limit_stiffness, tp.damping) for tp in a.tendon_props if tp.limit_stiffness > 0.0}
            if len(ks) > 1:
                raise NotImplementedError("all active tendons share one limit stiffness / damping")
            tk, td = next(iter(ks)) if ks else (0.0, 0.0)
            if obj is None:
                tend = []
            ext = engine.pack_model_ext(model, obj=obj, actors_per_env=apr, tendons=tend, tendon_k=tk, tendon_d=td)
        if ext is not None and hf_kw:
            raise NotImplementedError("multi-actor envs run on the ground plane")
        sim.engine = engine.Sim(model, len(sim.envs), dt=p.dt, substeps=p.substeps, gravity=(g.x, g.y, g.z), ground_mu=mu,
                                device=f"cuda:{sim.compute_device}", ext=ext, **hf_kw)
        poses = torch.tensor([[[q.p.x, q.p.y, q.p.z, q.r.x, q.r.y, q.r.z, q.r.w] for q in env_poses] for env_poses in sim.start_poses],
                             dtype=torch.float32)
        sim.engine.root_state.view(len(sim.envs), apr, 13)[:, :, 0:7] = poses.to(sim.engine.root_state.device)
        return True

    def simulate(self, sim):
        sim.engine.simulate()
        if sim.obj_force_set:       # applied forces act for one simulate() (the caller re-applies them every step, shadow_hand.py:708)
            sim.obj_force.zero_(); sim.obj_force_set = False
        sim.frame += 1

    def fetch_results(self, sim, wait):
        pass

    def get_frame_count(self, sim):
        return sim.frame

    def get_sim_params(self, sim):
        return sim.params

    def set_sim_params(self, sim, params):
        sim.params = params

    # ---- assets (ant.py:149-178, humanoid.py:152-171, cartpole.py:84-113)
    def load_asset(self, sim, root, file, options=None):
        o = options or AssetOptions()
        opts = BuildOptions(fix_base_link=o.fix_base_link, collapse_fixed_joints=o.collapse_fixed_joints,
                            replace_cylinder_with_capsule=o.replace_cylinder_with_capsule, armature=o.armature,
                            density=o.density, angular_damping=o.angular_damping, linear_damping=o.linear_damping,
                            max_angular_velocity=o.max_angular_velocity,
                            disable_gravity=o.disable_gravity, default_dof_drive_mode=o.default_dof_drive_mode,
                            # fixed-base arms meet objects, not just the ground: one more sphere per capsule
                            capsule_mid_spheres=1 if o.fix_base_link else 0)
        return _Asset(load_asset_file(root, file, opts), copy.copy(o))   # the caller may go on mutating `options` (shadow_hand.py:279-282)

    # procedural single-body assets (ball_balance.py:277 create_sphere, franka_cube_stack.py:223-245 create_box): one primitive,
    # mass = options.density x volume; usable as the free object of an env (the engine's rounded box covers all three)
    def _primitive(self, name, gtype, size, options):
        from ..importer.model import IRBody, IRGeom, build_model
        o = options or AssetOptions()
        g = IRGeom(name, gtype, np.zeros(3), np.eye(3), np.asarray(size, dtype=np.float64))
        g.density = float(o.density)
        body = IRBody(name=name, pos=np.zeros(3), R=np.eye(3), geoms=[g])
        opts = BuildOptions(fix_base_link=o.fix_base_link, density=o.density, angular_damping=o.angular_damping, linear_damping=o.linear_damping,
                            max_angular_velocity=o.max_angular_velocity, disable_gravity=o.disable_gravity)
        return _Asset(build_model(name, body, has_free_root=not o.fix_base_link, opts=opts), copy.copy(o))

    def create_box(self, sim, width, height, depth, options=None):
        from ..importer.model import GEOM_BOX
        return self._primitive("box", GEOM_BOX, [0.5 * width, 0.5 * height, 0.5 * depth], options)

    def create_sphere(self, sim, radius, options=None):
        from ..importer.model import GEOM_SPHERE
        return self._primitive("sphere", GEOM_SPHERE, [radius], options)

    def create_capsule(self, sim, radius, length, options=None):        # axis along x in gymapi; the object's frame is free, ours is z
        from ..importer.model import GEOM_CAPSULE
        return self._primitive("capsule", GEOM_CAPSULE, [radius, 0.5 * length], options)

    def get_asset_dof_count(self, asset):
        return asset.model.ndof

    def get_asset_rigid_body_count(self, asset):
        return asset.model.nb

    def get_asset_joint_count(self, asset):
        names = getattr(asset.model, "body_joint_names", None)
        return asset.model.ndof if not names else len(names) - 1          # one joint per non-root body (fixed ones included)

    def _joint_names(self, model):
        names = getattr(model, "body_joint_names", None)
        if not names:
            raise NotImplementedError("joint names: this compiled model was built before the importer recorded them; load the asset from its XML")
        return names

    def get_asset_joint_names(self, asset):
        return list(self._joint_names(asset.model)[1:])

    def get_asset_joint_dict(self, asset):
        """joint name -> index; joint k connects body k + 1 to its parent, so the index also addresses that body's row of a
        fixed-base Jacobian tensor (`jacobian[:, joint_dict['panda_hand_joint'], :, :7]`, franka_cube_stack.py:390-391)"""
        return {n: i for i, n in enumerate(self._joint_names(asset.model)[1:]) if n}

    def get_asset_rigid_shape_count(self, asset):
        return len(asset.model.geom_type)

    def get_asset_rigid_body_name(self, asset, i):
        return asset.model.body_names[i]

    def get_asset_rigid_body_names(self, asset):
        return list(asset.model.body_names)

    def get_asset_dof_names(self, asset):
        return list(asset.model.dof_names)

    def find_asset_dof_index(self, asset, name):
        return asset.model.dof_names.index(name)

    def find_asset_rigid_body_index(self, asset, name):
        return asset.model.body_names.index(name)

    def get_asset_actuator_count(self, asset):
        return len(asset.model.actuator_names)

    def get_asset_actuator_joint_name(self, asset, i):
        return asset.model.actuator_joint[i]

    def get_asset_actuator_properties(self, asset):
        m = asset.model
        return [types.SimpleNamespace(motor_effort=float(g), kp=float(k), lower_force_limit=float(fr[0]), upper_force_limit=float(fr[1]))
                for g, k, fr in zip(m.actuator_gear, m.actuator_kp, m.actuator_forcerange)]

    def get_asset_dof_properties(self, asset):
        m = asset.model
        dt = np.dtype([("hasLimits", "?"), ("lower", "f4"), ("upper", "f4"), ("driveMode", "i4"), ("velocity", "f4"),
                       ("effort", "f4"), ("stiffness", "f4"), ("damping", "f4"), ("friction", "f4"), ("armature", "f4")])
        p = np.zeros(m.ndof, dtype=dt)
        p["hasLimits"] = m.limited[1:] > 0
        p["lower"], p["upper"] = m.lower[1:], m.upper[1:]
        p["driveMode"] = m.drive_mode[1:]
        p["velocity"] = np.minimum(m.velocity[1:], 3e38); p["effort"] = np.minimum(m.effort[1:], 3e38)
        p["stiffness"], p["damping"], p["armature"] = m.kp[1:], m.kd[1:], m.armature[1:]
        return p

    # ---- tendons (shadow_hand.py:253-266)
    def get_asset_tendon_count(self, asset):
        return len(asset.tendon_props)

    def get_asset_tendon_name(self, asset, i):
        return asset.model.tendons[i]["name"]

    def get_asset_tendon_properties(self, asset):
        return asset.tendon_props

    def set_asset_tendon_properties(self, asset, props):
        asset.tendon_props = props

    def get_asset_rigid_shape_properties(self, asset):
        return asset.shape_props

    def set_asset_rigid_shape_properties(self, asset, props):
        asset.shape_props = props

    def create_asset_force_sensor(self, asset, body_idx, local_pose, props=None):
        asset.sensors.append((int(body_idx), local_pose))
        return len(asset.sensors) - 1

    # ---- envs / actors (ant.py:185-212)
    def create_env(self, sim, lower, upper, num_per_row):
        e = _Env(len(sim.envs))
        e.sim = sim
        sim.envs.append(e)
        return e

    def create_actor(self, env, asset, pose, name, group, filter, seg_id=0):
        sim = env.sim
        k = len(env.actors)
        if k == 0:
            if sim.asset is None:
                sim.asset = asset
            elif sim.asset is not asset:
                raise NotImplementedError("every env holds the same articulation as its first actor")
            sim.start_poses.append([])
        elif env.index == 0:
            sim.extra_assets.append(asset)
        elif k - 1 >= len(sim.extra_assets) or sim.extra_assets[k - 1] is not asset:
            raise NotImplementedError("every env holds the same actors in the same order")
        if env.index == 0 and filter <= 0 and getattr(asset, "model", None) is not None and getattr(asset.model, "ndof", 0) > 2:
            from .. import engine as _engine                 # filter 0: PhysX collides the actor's links with each other
            from ..importer.model import enable_self_collision, self_collision_supported
            if filter == 0 and k == 0 and self_collision_supported(asset.model):
                if not getattr(asset.model, "self_collide", False):
                    enable_self_collision(asset.model)
            else:                                            # four-chain kernels, asset-defined pairs (-1), later actors: said, not dropped
                _engine.warn_self_collision(f"actor '{name}'", f"create_actor(..., collision_filter={filter})")
        env.actors.append(name)
        env.actor_ids.append(sim.num_actors)            # sim-domain index: creation order (shadow_hand.py:356,369,376)
        sim.num_actors += 1
        sim.start_poses[env.index].append(Transform(Vec3(pose.p.x, pose.p.y, pose.p.z), Quat(pose.r.x, pose.r.y, pose.r.z, pose.r.w)))
        return k

    def begin_aggregate(self, *a):
        pass

    def end_aggregate(self, *a):
        pass

    def set_rigid_body_color(self, *a):
        pass

    def get_actor_dof_properties(self, env, actor):
        return self.get_asset_dof_properties(env.sim.asset)

    def set_actor_dof_properties(self, env, actor, props):
        m = env.sim.asset.model
        m.kp[1:] = props["stiffness"]; m.kd[1:] = props["damping"]
        m.drive_mode[1:] = props["driveMode"]
        return True

    def enable_actor_dof_force_sensors(self, env, actor):
        return True

    def find_actor_rigid_body_handle(self, env, actor, name):
        return env.sim.asset.model.body_names.index(name)

    def get_actor_index(self, env, actor, domain):
        return env.actor_ids[int(actor)] if domain == DOMAIN_SIM else int(actor)

    def get_actor_rigid_body_properties(self, env, actor):
        m = env.sim.asset.model if int(actor) == 0 else env.sim.extra_assets[int(actor) - 1].model
        return [types.SimpleNamespace(mass=float(m.mass[m.body_link[b]])) for b in range(m.nb)]

    def get_sim_actor_count(self, sim):
        return len(sim.envs) * (1 + len(sim.extra_assets))

    def get_actor_dof_count(self, env, actor):
        return env.sim.asset.model.ndof if int(actor) == 0 else 0

    def get_actor_rigid_body_count(self, env, actor):
        return env.sim.asset.model.nb if int(actor) == 0 else 1

    # name -> index maps of the articulation (body / DOF order = the tensors' order)
    def get_asset_rigid_body_dict(self, asset):
        return {n: i for i, n in enumerate(asset.model.body_names)}

    def get_asset_dof_dict(self, asset):
        return {n: i for i, n in enumerate(asset.model.dof_names)}

    def get_actor_rigid_body_dict(self, env, actor):
        return self.get_asset_rigid_body_dict(env.sim.asset)

    def get_actor_dof_dict(self, env, actor):
        return self.get_asset_dof_dict(env.sim.asset)

    def get_actor_joint_dict(self, env, actor):
        return self.get_asset_joint_dict(env.sim.asset)

    def get_actor_joint_names(self, env, actor):
        return self.get_asset_joint_names(env.sim.asset)

    def get_actor_joint_count(self, env, actor):
        return self.get_asset_joint_count(env.sim.asset)

    def get_actor_rigid_body_names(self, env, actor):
        return list(env.sim.asset.model.body_names)

    def get_actor_dof_names(self, env, actor):
        return list(env.sim.asset.model.dof_names)

    def find_actor_dof_handle(self, env, actor, name):
        return env.sim.asset.model.dof_names.index(name)

    def find_actor_dof_index(self, env, actor, name, domain):
        i = env.sim.asset.model.dof_names.index(name)
        return i + env.index * env.sim.asset.model.ndof if domain == DOMAIN_SIM else i

    def debug_print_asset(self, asset):
        m = asset.model
        print(f"asset: {m.nb} bodies {list(m.body_names)}, {m.ndof} dofs {list(m.dof_names)}")

    def get_sim_dof_count(self, sim):
        return sim.asset.model.ndof * len(sim.envs)

    def get_env_origin(self, env):
        return Vec3()

    # ---- state views (ant.py:78-95, humanoid.py:85-86, anymal_terrain.py:119)
    def acquire_actor_root_state_tensor(self, sim):
        return _Tensor(sim.engine.root_state)

    def acquire_dof_state_tensor(self, sim):
        return _Tensor(sim.engine.dof_state)

    def acquire_force_sensor_tensor(self, sim):
        return _Tensor(sim.engine.acquire(engine.T_FORCE_SENSOR))

    def acquire_dof_force_tensor(self, sim):
        return _Tensor(sim.engine.acquire(engine.T_DOF_FORCE))

    def acquire_rigid_body_state_tensor(self, sim):
        return _Tensor(sim.engine.acquire(engine.T_RIGID_BODY_STATE))

    def acquire_net_contact_force_tensor(self, sim):
        return _Tensor(sim.engine.acquire(engine.T_NET_CONTACT))

    # franka_cube_stack.py:388-392: `acquire_jacobian_tensor(sim, actor_name)`; one articulation per env here, so the name
    # only has to be an actor that was created
    def acquire_jacobian_tensor(self, sim, name):
        return _Tensor(sim.engine.acquire(engine.T_JACOBIAN))

    def acquire_mass_matrix_tensor(self, sim, name):
        return _Tensor(sim.engine.acquire(engine.T_MASS_MATRIX))

    def refresh_jacobian_tensors(self, sim):             # franka_cube_stack.py:439
        sim.engine.refresh_kinematic_tensors(jacobian=True, mass_matrix=False)
        return True

    def refresh_mass_matrix_tensors(self, sim):          # franka_cube_stack.py:440
        sim.engine.refresh_kinematic_tensors(jacobian=False, mass_matrix=True)
        return True

    def refresh_actor_root_state_tensor(self, sim):      # written in place by simulate
        return True

    refresh_dof_state_tensor = refresh_force_sensor_tensor = refresh_dof_force_tensor = refresh_actor_root_state_tensor
    refresh_net_contact_force_tensor = refresh_actor_root_state_tensor

    def refresh_rigid_body_state_tensor(self, sim):
        sim.engine.refresh_rigid_body_state()
        return True

    # ---- writes (ant.py:265-285)
    def set_dof_actuation_force_tensor(self, sim, t):
        sim.engine.dof_actuation.view(-1).copy_(t.view(-1))
        return True

    def set_dof_actuation_force_tensor_indexed(self, sim, t, idx, n):        # idx = actor indices (DOMAIN_SIM), like the other *_indexed setters
        nd = sim.asset.model.ndof
        i = idx[:n].long() // (1 + len(sim.extra_assets))
        sim.engine.dof_actuation.view(-1, nd)[i] = t.view(-1, nd)[i]
        return True

    def set_dof_position_target_tensor(self, sim, t):
        sim.engine.dof_target.view(-1).copy_(t.view(-1))
        return True

    def set_dof_position_target_tensor_indexed(self, sim, t, idx, n):       # shadow_hand.py:646-648; idx = actor indices
        nd = sim.asset.model.ndof
        i = idx[:n].long() // (1 + len(sim.extra_assets))
        sim.engine.dof_target.view(-1, nd)[i] = t.view(-1, nd)[i]
        return True

    def apply_rigid_body_force_tensors(self, sim, forces=None, torques=None, space=ENV_SPACE):   # shadow_hand.py:708
        """Forces at the centre of mass for the next simulate().  The engine applies them to the simulated free object of an
        env (the body the reference pushes); a non-zero force on an articulation link or any torque raises."""
        if torques is not None and bool((torques != 0).any()):
            raise NotImplementedError("apply_rigid_body_force_tensors: torques are not applied by the engine")
        if forces is None:
            return True
        eng = sim.engine
        n, nb = eng.num_envs, sim.asset.model.nb
        f = forces.view(n, -1, 3)
        if f.shape[1] != nb + len(sim.extra_assets):
            raise ValueError("apply_rigid_body_force_tensors: expected one row per rigid body of the sim")
        has_obj = eng.actors_per_env > 1 and len(sim.extra_assets) > 0 and not sim.extra_assets[0].options.disable_gravity
        others = f.clone()
        if has_obj:
            others[:, nb] = 0
        if bool((others != 0).any()):
            raise NotImplementedError("apply_rigid_body_force_tensors: only the free object of an env takes external forces")
        if not has_obj:
            return True
        fo = f[:, nb].to(torch.float32)
        if space != LOCAL_SPACE:                                # env / global axes -> the object's own frame
            q = eng.root_state.view(n, eng.actors_per_env, 13)[:, 1, 3:7]
            qv, qw = q[:, :3], q[:, 3:4]
            a = fo * (2.0 * qw * qw - 1.0); b = torch.cross(qv, fo, dim=-1) * qw * 2.0
            c = qv * (qv * fo).sum(-1, keepdim=True) * 2.0
            fo = a - b + c                                      # quat_rotate_inverse, torch_jit_utils.py:72-81
        if sim.obj_force is None:
            sim.obj_force = eng._bind(engine.T_OBJ_FORCE, torch.zeros(n, 3, dtype=torch.float32, device=eng.root_state.device))
        sim.obj_force.copy_(fo); sim.obj_force_set = True
        return True

    def set_actor_root_state_tensor(self, sim, t):
        if t.data_ptr() != sim.engine.root_state.data_ptr():
            sim.engine.root_state.copy_(t.view_as(sim.engine.root_state))
        return True

    def set_actor_root_state_tensor_indexed(self, sim, t, idx, n):
        if t.data_ptr() != sim.engine.root_state.data_ptr():
            i = idx[:n].long()
            sim.engine.root_state[i] = t.view_as(sim.engine.root_state)[i]
        return True

    def set_dof_state_tensor(self, sim, t):
        if t.data_ptr() != sim.engine.dof_state.data_ptr():
            sim.engine.dof_state.copy_(t.view_as(sim.engine.dof_state))
        return True

    def set_dof_state_tensor_indexed(self, sim, t, idx, n):
        if t.data_ptr() != sim.engine.dof_state.data_ptr():
            nd = sim.asset.model.ndof
            i = idx[:n].long() // (1 + len(sim.extra_assets))     # actor index of the articulation -> env
            sim.engine.dof_state.view(-1, nd, 2)[i] = t.view(-1, nd, 2)[i]
        return True

    # ---- viewer (headless only)
    def create_viewer(self, sim, props):
        return None

    def viewer_camera_look_at(self, *a):
        pass

    def add_lines(self, *a):             # debug drawing (ant.py:307-321): headless
        pass

    def clear_lines(self, *a):
        pass


_GYM = Gym()


def acquire_gym():
    """Process-wide singleton (vec_task.py:247)."""
    return _GYM
