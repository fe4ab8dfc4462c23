"""Articulation model: the compiled, flat description of one actor asset that the CUDA engine,
the C oracle and the `gym.get_asset_*` queries all read.

The reference's importer lives inside the closed `isaacgym` binary (SURVEY.md §2 row 14), so the
semantics below are restated from the asset files themselves and the call sites that query them
(`isaacgymenvs/tasks/ant.py:149-212`, `humanoid.py:152-207`, `cartpole.py:84-113`).

Internal convention ("links"): every DOF is its own 1-DOF link (hinge or slide).  A body carrying
several joints (MJCF compound joints, `nv_humanoid.xml:53-54`) becomes a chain of links of which
only the last has mass; jointless child bodies are welded into their parent's link but stay
visible as *bodies* (the reference counts them: Humanoid has 16 rigid bodies, `humanoid.py:158`).
Link frame i: origin at the joint anchor, axes = the body's axes.  DOF k drives link k+1.
"""
from dataclasses import dataclass, field
import json
import numpy as np

from . import rot

JOINT_HINGE, JOINT_SLIDE = 0, 1
GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX, GEOM_CYLINDER, GEOM_ELLIPSOID = 0, 1, 2, 3, 4
DRIVE_NONE, DRIVE_POS, DRIVE_VEL, DRIVE_EFFORT = 0, 1, 2, 3  # gymapi.DOF_MODE_* order


# --------------------------------------------------------------------------- intermediate tree
@dataclass
class IRJoint:
    name: str
    jtype: int
    axis: np.ndarray
    anchor: np.ndarray            # in the body frame
    lower: float = 0.0
    upper: float = 0.0
    limited: bool = False
    armature: float = 0.0
    damping: float = 0.0
    stiffness: float = 0.0
    effort: float = 1e30          # URDF <limit effort>
    velocity: float = 1e30
    friction: float = 0.0


@dataclass
class IRGeom:
    name: str
    gtype: int
    pos: np.ndarray
    R: np.ndarray
    size: np.ndarray              # sphere (r,), capsule/cylinder (r, half_len) along local z, box half-sizes
    density: float = 1000.0
    mass: float = -1.0            # explicit geom mass overrides density
    friction: float = 1.0
    collide: bool = True


class UnmodelledGeometryWarning(UserWarning):
    """Collision geometry of an asset that the importer cannot turn into a primitive (triangle / convex meshes, SURVEY.md 8f rank
    4): the bodies it belongs to do not collide through it.  Emitted once per import; Model.unmodelled_geoms lists them."""


@dataclass
class IRBody:
    name: str
    pos: np.ndarray
    R: np.ndarray
    joints: list = field(default_factory=list)
    geoms: list = field(default_factory=list)
    inertial: tuple = None        # (mass, com(3), I_com 3x3 in body axes) or None -> from geoms
    children: list = field(default_factory=list)
    sites: dict = field(default_factory=dict)
    collapsed: bool = False       # jointless body merged away (URDF collapse_fixed_joints)
    parent_joint: str = ""        # name of the joint to the parent body (URDF: every non-root link has exactly one, fixed ones included)
    skipped_geoms: list = field(default_factory=list)   # collision geometry the importer has no primitive for (meshes): names
    extra_parts: list = field(default_factory=list)     # (mass, com, inertia 3x3 about it) of such geometry, body frame: counted when the body has no <inertial>


def geom_mass_inertia(g):
    """Mass, inertia (3x3 about the geom centre, geom axes) of a primitive of uniform density."""
    t, s = g.gtype, g.size
    if t == GEOM_SPHERE:
        r = s[0]
        v = 4.0 / 3.0 * np.pi * r ** 3
        m = g.mass if g.mass >= 0 else g.density * v
        return m, np.eye(3) * (0.4 * m * r * r)
    if t == GEOM_CAPSULE:
        r, l = s[0], s[1]
        vc, vs = np.pi * r * r * 2 * l, 4.0 / 3.0 * np.pi * r ** 3
        m = g.mass if g.mass >= 0 else g.density * (vc + vs)
        mc, ms = m * vc / (vc + vs), m * vs / (vc + vs)
        izz = mc * r * r / 2 + ms * 0.4 * r * r
        ixx = mc * (r * r / 4 + l * l / 3) + ms * (0.4 * r * r + l * l + 0.75 * l * r)
        return m, np.diag([ixx, ixx, izz])
    if t == GEOM_CYLINDER:
        r, l = s[0], s[1]
        m = g.mass if g.mass >= 0 else g.density * np.pi * r * r * 2 * l
        return m, np.diag([m * (3 * r * r + 4 * l * l) / 12] * 2 + [m * r * r / 2])
    if t == GEOM_BOX:
        a, b, c = s
        m = g.mass if g.mass >= 0 else g.density * 8 * a * b * c
        return m, np.diag([m * (b * b + c * c) / 3, m * (a * a + c * c) / 3, m * (a * a + b * b) / 3])
    if t == GEOM_ELLIPSOID:
        a, b, c = s
        m = g.mass if g.mass >= 0 else g.density * 4.0 / 3.0 * np.pi * a * b * c
        return m, np.diag([m * (b * b + c * c) / 5, m * (a * a + c * c) / 5, m * (a * a + b * b) / 5])
    raise ValueError(f"geom type {t}")


def combine_inertia(parts):
    """parts: list of (m, com(3), I_com(3x3)) in one frame -> (m, com, I_com)."""
    M = sum(p[0] for p in parts)
    if M <= 0:
        return 0.0, np.zeros(3), np.zeros((3, 3))
    c = sum(p[0] * p[1] for p in parts) / M
    I = np.zeros((3, 3))
    for m, pc, Ic in parts:
        d = pc - c
        I += Ic + m * ((d @ d) * np.eye(3) - np.outer(d, d))
    return M, c, I


# --------------------------------------------------------------------------- compiled model
@dataclass
class Model:
    name: str = ""
    root_fixed: bool = False
    # links
    parent: np.ndarray = None     # (nl,) int, -1 for the root
    jtype: np.ndarray = None      # (nl,) int, -1 for the root
    axis: np.ndarray = None       # (nl,3) unit, link frame
    lpos: np.ndarray = None       # (nl,3) link origin in the parent link frame at q=0
    lquat: np.ndarray = None      # (nl,4) xyzw link orientation in the parent link frame at q=0
    mass: np.ndarray = None
    com: np.ndarray = None        # (nl,3) link frame
    inertia: np.ndarray = None    # (nl,6) xx,yy,zz,xy,xz,yz about the COM, link axes
    # per-DOF (index = link index, entry 0 unused)
    armature: np.ndarray = None
    damping: np.ndarray = None
    stiffness: np.ndarray = None
    lower: np.ndarray = None
    upper: np.ndarray = None
    limited: np.ndarray = None
    effort: np.ndarray = None
    velocity: np.ndarray = None
    kp: np.ndarray = None
    kd: np.ndarray = None
    drive_mode: np.ndarray = None
    limit_k: np.ndarray = None    # joint-limit penalty spring / damper (DESIGN.md "joint limits")
    limit_d: np.ndarray = None
    # bodies (public numbering)
    body_names: list = None
    body_link: np.ndarray = None  # (nb,)
    body_pos: np.ndarray = None   # (nb,3) body frame in its link frame
    body_quat: np.ndarray = None  # (nb,4)
    dof_names: list = None
    # collision primitives (for queries / non-plane contact) and plane contact points
    geom_names: list = None
    geom_type: np.ndarray = None
    geom_link: np.ndarray = None
    geom_body: np.ndarray = None
    geom_pos: np.ndarray = None   # (ng,3) link frame
    geom_quat: np.ndarray = None
    geom_size: np.ndarray = None  # (ng,3)
    geom_friction: np.ndarray = None
    cp_link: np.ndarray = None    # (ncp,) contact spheres tested against plane / heightfield
    cp_pos: np.ndarray = None     # (ncp,3) link frame
    cp_radius: np.ndarray = None
    cp_mu: np.ndarray = None
    cp_body: np.ndarray = None
    # box primitives kept as boxes (another body's corner points are tested against them: hand-object contact)
    box_link: np.ndarray = None   # (nbx,)
    box_body: np.ndarray = None
    box_pos: np.ndarray = None    # (nbx,3) link frame
    box_quat: np.ndarray = None   # (nbx,4)
    box_half: np.ndarray = None   # (nbx,3)
    # force sensors (body frame), actuators, tendons
    sensor_body: np.ndarray = None
    sensor_pos: np.ndarray = None
    sensor_quat: np.ndarray = None
    actuator_names: list = None
    actuator_joint: list = None   # dof names
    actuator_gear: np.ndarray = None
    actuator_kp: np.ndarray = None
    actuator_forcerange: np.ndarray = None  # (na,2)
    actuator_kind: list = None    # 'motor' | 'position'
    tendons: list = None          # [{name, dofs:[..], coefs:[..], range:[lo,hi], limited}]
    # penalty-contact parameters (see DESIGN.md "contact model")
    contact_kn: float = 0.0
    contact_cn: float = 0.0
    contact_vs: float = 0.02
    gravity_on: bool = True
    # AssetOptions.angular_damping / linear_damping / max_angular_velocity (humanoid.py:153-154, anymal_terrain.py:225-226):
    # every link's COM twist is damped with acceleration -d * v (a wrench -d_a Ic w, -d_l m v_c on the link), the base's
    # angular speed is clamped after integration (DESIGN.md "physics model")
    angular_damping: float = 0.0
    linear_damping: float = 0.0
    max_angular_velocity: float = 64.0
    # self-collision (create_actor collision filter 0: humanoid.py:194, anymal_terrain.py:282): set by enable_self_collision()
    self_collide: bool = False
    self_pairs: np.ndarray = None        # (ncp, ncp) uint8, 1 = the ordered pair of contact spheres may collide
    self_kn: float = 0.0
    self_cn: float = 0.0
    self_mu: float = 1.0
    build_options: dict = None           # the BuildOptions this model was compiled with (checked when a committed blob stands in for the XML)
    default_root_pos: np.ndarray = None  # body pose from the file (Ant overrides it at create_actor)
    default_root_quat: np.ndarray = None

    @property
    def nl(self):
        return len(self.parent)

    @property
    def ndof(self):
        return self.nl - 1

    @property
    def nb(self):
        return len(self.body_names)

    def total_mass(self):
        return float(np.sum(self.mass))

    def depth(self):
        d = np.zeros(self.nl, dtype=int)
        for i in range(1, self.nl):
            d[i] = d[self.parent[i]] + 1
        return d

    # ---- (de)serialisation: committed under assets/compiled/*.json so the GPU box, which has no
    # the reference checkout, can build the same model
    def to_json(self):
        out = {}
        for k, v in self.__dict__.items():
            if isinstance(v, np.ndarray):
                out[k] = {"__nd__": v.tolist(), "dtype": str(v.dtype)}
            else:
                out[k] = v
        return json.dumps(out, indent=None, separators=(",", ":"))

    @staticmethod
    def from_json(s):
        d = json.loads(s)
        m = Model()
        for k, v in d.items():
            if isinstance(v, dict) and "__nd__" in v:
                v = np.array(v["__nd__"], dtype=v["dtype"])
                if v.ndim == 1 and v.size == 0:
                    pass
            setattr(m, k, v)
        return m


def enable_self_collision(m: "Model", kappa=0.5, zeta=0.5, mu=1.0, samples=4096, margin=0.10):
    """create_actor(..., collision_filter=0): links of the articulation collide with each other.  Candidate pairs = contact
    spheres on links that are not joint neighbours (same link, or parent / child through massless intermediate links of a
    compound joint, never collide -- PhysX filters those too), and whose spheres do not already overlap in the reference
    pose q = 0 (adjacent capsules of a chain share end spheres by construction).
    Gains PER PAIR from the reduced mass of the two links and the sub-step h: kn = kappa m_red / h^2, cn = zeta m_red / h
    (self_kn = kappa, self_cn = zeta are dimensionless).  The coupling is block-Jacobi -- each link implicit in its own
    acceleration, explicit in the partner's velocity -- and that half-explicit scheme is stable only while h^2 kn / m and
    h cn / m stay below ~1 for the lighter body.  Gains tied to the ACTOR's mass (as the ground contact's are) were measured
    first: fine under random torques, but persistent bang-bang actuation -- what a learner produces -- blew joint speeds up to
    1e5 rad/s (243 blow-ups in 600 steps x 512 envs; none at kappa = zeta = 0.5, 3-4 at kappa = 1).  The price is a soft
    contact: under full-scale random torques 23 % of sampled states still overlap by > 1 cm (53 % without, deepest 5.6 vs 11.4 cm).
    friction mu = the MJCF default geom friction under PhysX's average combine mode."""
    ncp = len(m.cp_link)
    carrier = set(int(l) for l in m.body_link)

    def up(l):
        l = int(m.parent[l])
        while l >= 0 and l not in carrier:
            l = int(m.parent[l])
        return l
    link = np.array([int(l) for l in m.cp_link])
    # spheres are attached to links; a massless intermediate link carries none, so "neighbour" is decided on carrying links
    def carrying(l):
        while l >= 0 and l not in carrier:
            l = int(m.parent[l])
        return l
    cl = np.array([carrying(int(l)) for l in link])
    anc = np.array([up(int(l)) if l >= 0 else -1 for l in cl])
    # reference pose: world centres at q = 0 (root at the origin)
    from . import rot
    nl = m.nl
    Rw = [np.eye(3)] * nl; pw = [np.zeros(3)] * nl
    for i in range(1, nl):
        pa = int(m.parent[i])
        Rw[i] = Rw[pa] @ rot.quat_to_mat(m.lquat[i]); pw[i] = pw[pa] + Rw[pa] @ np.asarray(m.lpos[i], float)
    wc = np.array([pw[link[n]] + Rw[link[n]] @ np.asarray(m.cp_pos[n], float) for n in range(ncp)])
    rad = np.asarray(m.cp_radius, float)
    pairs = np.zeros((ncp, ncp), np.uint8)
    for a in range(ncp):
        for b in range(ncp):
            if cl[a] == cl[b] or anc[a] == cl[b] or anc[b] == cl[a]:
                continue
            if np.linalg.norm(wc[a] - wc[b]) < rad[a] + rad[b]:           # overlapping by construction
                continue
            pairs[a, b] = 1
    # reachability: a pair whose spheres stay more than `margin` apart in every joint configuration inside the limits can be
    # dropped without changing the physics (a Humanoid's foot never meets its head).  Decided from `samples` random
    # configurations (fixed seed) with a generous margin; most of the per-step cost is proportional to the pairs kept.
    if samples > 0 and pairs.any():
        rng = np.random.default_rng(12345)
        lo = np.where(np.asarray(m.limited[1:]) > 0, np.asarray(m.lower[1:], float), -np.pi)
        hi = np.where(np.asarray(m.limited[1:]) > 0, np.asarray(m.upper[1:], float), np.pi)
        q = rng.uniform(lo, hi, size=(samples, nl - 1))
        q[: samples // 4] = np.where(rng.random((samples // 4, nl - 1)) < 0.5, lo, hi)      # a quarter at the corners of the limit box
        R = np.zeros((samples, nl, 3, 3)); P = np.zeros((samples, nl, 3)); R[:, 0] = np.eye(3)
        for i in range(1, nl):
            pa = int(m.parent[i])
            Rl = rot.quat_to_mat(m.lquat[i]); ax = np.asarray(m.axis[i], float)
            if int(m.jtype[i]) == JOINT_HINGE:
                K = np.array([[0, -ax[2], ax[1]], [ax[2], 0, -ax[0]], [-ax[1], ax[0], 0]])
                ang = q[:, i - 1][:, None, None]
                Rj = np.eye(3)[None] + np.sin(ang) * K[None] + (1 - np.cos(ang)) * (K @ K)[None]
                R[:, i] = R[:, pa] @ (Rl[None] @ Rj)
                P[:, i] = P[:, pa] + R[:, pa] @ np.asarray(m.lpos[i], float)
            else:
                R[:, i] = R[:, pa] @ Rl[None]
                P[:, i] = P[:, pa] + R[:, pa] @ np.asarray(m.lpos[i], float) + (R[:, i] @ ax) * q[:, i - 1][:, None]
        W = np.stack([P[:, link[n]] + R[:, link[n]] @ np.asarray(m.cp_pos[n], float) for n in range(ncp)], 1)   # (samples, ncp, 3)
        gap = np.full((ncp, ncp), np.inf)
        for a in range(ncp):
            d = np.linalg.norm(W[:, a:a + 1] - W, axis=-1) - (rad[a] + rad)[None]
            gap[a] = d.min(0)
        pairs = (pairs.astype(bool) & (gap < margin)).astype(np.uint8)
        pairs = (pairs | pairs.T).astype(np.uint8)
    m.self_pairs = pairs
    m.self_kn = float(kappa)
    m.self_cn = float(zeta)
    m.self_mu = float(mu)
    m.self_collide = True
    return m


def self_collision_supported(m: "Model"):
    """Which models the engine's link-link contact covers: the generic sub-step, <= 64 contact spheres, <= 32 links.  A free base
    with four identical hinge chains (Ant, ANYmal) runs on the four-chain kernels, which do not carry it: such a model keeps
    its speed and says so (engine.warn_self_collision) instead."""
    if len(m.cp_link) > 64 or m.nl > 32:
        return False
    if not m.root_fixed and m.ndof in (8, 12):
        kids = [i for i in range(1, m.nl) if m.parent[i] == 0]
        if len(kids) == 4 and all(int(j) == JOINT_HINGE for j in m.jtype[1:]):
            return False
    return True


def finalize_limits(m: "Model", pen_rad=0.02, tau_s=0.01):
    """Joint-limit penalty gains: the strongest torque the DOF can see (actuator gear / URDF effort,
    at least 1) is met at `pen_rad` of penetration; damping time constant `tau_s`.  The terms are
    integrated implicitly, so the choice affects stiffness, not stability."""
    strength = np.ones(m.nl)
    for k, jn in enumerate(m.actuator_joint or []):
        li = m.dof_names.index(jn) + 1
        g = abs(m.actuator_gear[k]) if m.actuator_kind[k] == "motor" else abs(m.actuator_forcerange[k][1])
        if g < 1e29:
            strength[li] = max(strength[li], g)
    eff = np.where(m.effort < 1e29, m.effort, 0.0)
    strength = np.maximum(strength, eff)
    scale = np.where(m.jtype == JOINT_SLIDE, 10.0, 1.0)   # slide limits: N/m, stiffer per unit
    m.limit_k = strength / pen_rad * scale
    m.limit_d = m.limit_k * tau_s
    m.limit_k[0] = m.limit_d[0] = 0.0


@dataclass
class BuildOptions:
    """Subset of gymapi.AssetOptions that changes the compiled model (SURVEY.md §8b 'assets')."""
    fix_base_link: bool = False
    collapse_fixed_joints: bool = False
    replace_cylinder_with_capsule: bool = False
    armature: float = 0.0             # added to every DOF (AssetOptions.armature)
    density: float = 1000.0           # used when a body has neither <inertial> nor a geom density
    angular_damping: float = 0.0
    linear_damping: float = 0.0
    max_angular_velocity: float = 64.0 # AssetOptions default (rad/s)
    disable_gravity: bool = False
    default_dof_drive_mode: int = DRIVE_NONE
    capsule_mid_spheres: int = 0       # extra contact spheres along a capsule's axis (hands: the cylinder part must touch objects too)
    contact_kn_per_kg: float = 2000.0  # DESIGN.md: kn = 2000 s^-2 * actor mass
    contact_zeta: float = 1.0


def build_model(name, root: IRBody, has_free_root: bool, opts: BuildOptions) -> Model:
    """Flatten an IR body tree (file order DFS = the reference's DOF/body order) into a Model."""
    L = dict(parent=[], jtype=[], axis=[], lpos=[], lquat=[], parts=[], jref=[])
    bodies = dict(names=[], link=[], pos=[], quat=[], joint=[])
    geoms = []
    sites = {}
    skipped = []

    def new_link(parent, jt, axis, lpos, R, j):
        L["parent"].append(parent); L["jtype"].append(jt)
        L["axis"].append(np.zeros(3) if axis is None else np.asarray(axis, float) / np.linalg.norm(axis))
        L["lpos"].append(np.asarray(lpos, float)); L["lquat"].append(rot.mat_to_quat(R))
        L["parts"].append([]); L["jref"].append(j)
        return len(L["parent"]) - 1

    def visit(b: IRBody, link, p_lb, R_lb, is_root, parent_bi=-1):
        # (p_lb, R_lb): pose of b's *parent body frame* expressed in link `link`
        if is_root:
            li = new_link(-1, -1, None, np.zeros(3), np.eye(3), None)
            p_b, R_b = np.zeros(3), np.eye(3)
        else:
            p0 = p_lb + R_lb @ b.pos          # body frame at q=0, in `link`
            R0 = R_lb @ b.R
            if b.joints:
                li, prev_anchor = link, None
                for k, j in enumerate(b.joints):
                    if k == 0:
                        li = new_link(link, j.jtype, j.axis, p0 + R0 @ j.anchor, R0, j)
                    else:
                        li = new_link(li, j.jtype, j.axis, j.anchor - prev_anchor, np.eye(3), j)
                    prev_anchor = j.anchor
                p_b, R_b = -prev_anchor, np.eye(3)
            else:
                li, p_b, R_b = link, p0, R0
        if b.collapsed and not b.joints and not is_root:
            bi = parent_bi
        else:
            bodies["names"].append(b.name); bodies["link"].append(li)
            bodies["pos"].append(p_b); bodies["quat"].append(rot.mat_to_quat(R_b))
            # the joint this body hangs on: a URDF link's one parent joint; an MJCF body's last joint (the one whose link carries it)
            bodies["joint"].append("" if is_root else (b.parent_joint or (b.joints[-1].name if b.joints else "")))
            bi = len(bodies["names"]) - 1
        skipped.extend(f"{b.name}:{g}" for g in b.skipped_geoms)
        # inertia of this body, expressed in link li
        if b.inertial is not None:
            m, c, I = b.inertial
            parts = [(m, np.asarray(c, float), np.asarray(I, float))]
        else:
            parts = []
            for g in b.geoms:
                m, Ig = geom_mass_inertia(g)
                parts.append((m, g.pos, g.R @ Ig @ g.R.T))
            parts.extend(b.extra_parts)
        for m, c, I in parts:
            L["parts"][li].append((m, p_b + R_b @ c, R_b @ I @ R_b.T))
        for g in b.geoms:
            if g.collide:
                geoms.append((g, li, bi, p_b + R_b @ g.pos, R_b @ g.R))
        for sname, spos in b.sites.items():
            sites[sname] = (bi, spos)
        for ch in b.children:
            visit(ch, li, p_b, R_b, False, bi)

    visit(root, -1, np.zeros(3), np.eye(3), True)

    nl = len(L["parent"])
    m = Model(name=name, root_fixed=(opts.fix_base_link or not has_free_root))
    m.parent = np.array(L["parent"], dtype=np.int32)
    m.jtype = np.array(L["jtype"], dtype=np.int32)
    m.axis = np.array(L["axis"]); m.lpos = np.array(L["lpos"]); m.lquat = np.array(L["lquat"])
    mass, com, inertia = np.zeros(nl), np.zeros((nl, 3)), np.zeros((nl, 6))
    for i in range(nl):
        M, c, I = combine_inertia(L["parts"][i])
        mass[i], com[i], inertia[i] = M, c, rot.mat_to_sym6(I)
    m.mass, m.com, m.inertia = mass, com, inertia

    def jattr(f, default=0.0):
        return np.array([default if j is None else getattr(j, f) for j in L["jref"]], dtype=np.float64)
    m.armature = jattr("armature") + np.where(m.jtype >= 0, opts.armature, 0.0)
    m.damping, m.stiffness = jattr("damping"), jattr("stiffness")
    m.lower, m.upper = jattr("lower"), jattr("upper")
    m.limited = np.array([0 if j is None else int(j.limited) for j in L["jref"]], dtype=np.int32)
    m.effort, m.velocity = jattr("effort", 1e30), jattr("velocity", 1e30)
    m.kp, m.kd = np.zeros(nl), np.zeros(nl)
    m.drive_mode = np.full(nl, opts.default_dof_drive_mode, dtype=np.int32)
    m.dof_names = [j.name for j in L["jref"][1:]]
    m.body_names = bodies["names"]
    m.body_joint_names = bodies["joint"]        # per body: the joint to its parent ("" for the root / unnamed): gym.get_actor_joint_dict
    m.unmodelled_geoms = skipped
    if skipped:
        import warnings
        warnings.warn(f"{name}: {len(skipped)} collision geometr{'y' if len(skipped) == 1 else 'ies'} without a primitive (meshes) skipped -- "
                      f"{', '.join(skipped[:6])}{' ...' if len(skipped) > 6 else ''}: those bodies do not collide through them; "
                      "their mass properties, where the asset gives none, come from the volume the mesh encloses (DESIGN.md section 7)", UnmodelledGeometryWarning, stacklevel=3)
    m.body_link = np.array(bodies["link"], dtype=np.int32)
    m.body_pos, m.body_quat = np.array(bodies["pos"]), np.array(bodies["quat"])

    # collision primitives + plane contact points
    gt, gl, gb, gp, gq, gs, gf, gn = [], [], [], [], [], [], [], []
    cps = []
    boxes = []
    for g, li, bi, p, R in geoms:
        t = g.gtype
        if t == GEOM_CYLINDER and opts.replace_cylinder_with_capsule:
            t = GEOM_CAPSULE
        size = np.zeros(3); size[:len(g.size)] = g.size
        gt.append(t); gl.append(li); gb.append(bi); gp.append(p); gq.append(rot.mat_to_quat(R))
        gs.append(size); gf.append(g.friction); gn.append(g.name)
        z = R[:, 2]
        if t == GEOM_SPHERE:
            cps.append((li, bi, p, size[0], g.friction))
        elif t in (GEOM_CAPSULE, GEOM_CYLINDER):
            cps.append((li, bi, p - z * size[1], size[0], g.friction))
            cps.append((li, bi, p + z * size[1], size[0], g.friction))
            for k in range(opts.capsule_mid_spheres):
                f = (k + 1) / (opts.capsule_mid_spheres + 1) * 2 - 1
                cps.append((li, bi, p + z * size[1] * f, size[0], g.friction))
        elif t == GEOM_BOX:
            if np.min(size) > 2e-3:
                boxes.append((li, bi, p, rot.mat_to_quat(R), size.copy()))
            for sx in (-1, 1):
                for sy in (-1, 1):
                    for sz in (-1, 1):
                        cps.append((li, bi, p + R @ (size * np.array([sx, sy, sz])), 0.0, g.friction))
        elif t == GEOM_ELLIPSOID:
            cps.append((li, bi, p, float(np.min(size)), g.friction))
    # drop contact spheres wholly inside another contact sphere of the same link (e.g. the Ant's
    # aux-capsule ends at the torso centre, nv_ant.xml:42-45) and exact duplicates
    keep = []
    for a, ca in enumerate(cps):
        inside = False
        for b_, cb in enumerate(cps):
            if a == b_ or ca[0] != cb[0]:
                continue
            d = np.linalg.norm(ca[2] - cb[2])
            if d + ca[3] <= cb[3] + 1e-12 and (ca[3] < cb[3] or a > b_):
                inside = True
                break
        if not inside:
            keep.append(ca)
    # a child's sphere centred on its own hinge anchor coincides -- in every configuration -- with a
    # parent sphere of the same radius at that anchor (capsule chains: nv_ant.xml:42-52): keep the parent's
    parent_of = L["parent"]
    dedup = []
    for ca in keep:
        li = ca[0]
        drop = False
        if li > 0 and L["jtype"][li] == JOINT_HINGE and np.linalg.norm(ca[2]) < 1e-9:
            for cb in keep:
                if cb[0] == parent_of[li] and abs(cb[3] - ca[3]) < 1e-12 and np.linalg.norm(cb[2] - L["lpos"][li]) < 1e-9:
                    drop = True
                    break
        if not drop:
            dedup.append(ca)
    keep = dedup
    m.geom_names = gn
    m.geom_type = np.array(gt, dtype=np.int32); m.geom_link = np.array(gl, dtype=np.int32)
    m.geom_body = np.array(gb, dtype=np.int32)
    m.geom_pos = np.array(gp).reshape(-1, 3); m.geom_quat = np.array(gq).reshape(-1, 4)
    m.geom_size = np.array(gs).reshape(-1, 3); m.geom_friction = np.array(gf, dtype=np.float64)
    m.cp_link = np.array([c[0] for c in keep], dtype=np.int32)
    m.cp_body = np.array([c[1] for c in keep], dtype=np.int32)
    m.cp_pos = np.array([c[2] for c in keep]).reshape(-1, 3)
    m.cp_radius = np.array([c[3] for c in keep], dtype=np.float64)
    m.cp_mu = np.array([c[4] for c in keep], dtype=np.float64)

    m.box_link = np.array([b[0] for b in boxes], dtype=np.int32); m.box_body = np.array([b[1] for b in boxes], dtype=np.int32)
    m.box_pos = np.array([b[2] for b in boxes]).reshape(-1, 3); m.box_quat = np.array([b[3] for b in boxes]).reshape(-1, 4)
    m.box_half = np.array([b[4] for b in boxes]).reshape(-1, 3)
    m.sensor_body = np.zeros(0, dtype=np.int32)
    m.sensor_pos = np.zeros((0, 3)); m.sensor_quat = np.zeros((0, 4))
    m.actuator_names, m.actuator_joint, m.actuator_kind = [], [], []
    m.actuator_gear = np.zeros(0); m.actuator_kp = np.zeros(0); m.actuator_forcerange = np.zeros((0, 2))
    m.tendons = []
    M = m.total_mass()
    m.contact_kn = opts.contact_kn_per_kg * M
    m.contact_cn = 2.0 * opts.contact_zeta * np.sqrt(m.contact_kn * M / 4.0)
    m.gravity_on = not opts.disable_gravity
    m.angular_damping, m.linear_damping = float(opts.angular_damping), float(opts.linear_damping)
    m.max_angular_velocity = float(opts.max_angular_velocity)
    m.build_options = {k: (float(v) if isinstance(v, float) else int(v) if isinstance(v, (bool, int)) else v) for k, v in opts.__dict__.items()}
    m.default_root_pos = np.asarray(root.pos, float)
    m.default_root_quat = rot.mat_to_quat(root.R)
    return m
