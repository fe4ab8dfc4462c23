"""MJCF -> IR body tree -> Model.

Only the MJCF features the five BASELINE assets use are implemented (SURVEY.md §7 hard part 3):
`<compiler angle inertiafromgeom>`, nested `<default class>` + `childclass`/`class`, `<include>`,
`<body pos quat euler>`, `<freejoint>` / `<joint type=hinge|slide|free>`, several joints per body,
`<geom type=sphere|capsule|box|cylinder|ellipsoid fromto size pos quat euler density mass friction>`,
`<inertial pos quat mass diaginertia|fullinertia>`, `<actuator><motor|position>`,
`<tendon><fixed>`.  Semantics follow the MuJoCo XML reference (published format), not any code in
the reference checkout: the reference parses these files inside the closed isaacgym binary.
"""
import os
import xml.etree.ElementTree as ET
import numpy as np

from . import rot
from .model import (IRBody, IRGeom, IRJoint, BuildOptions, build_model, finalize_limits, JOINT_HINGE, JOINT_SLIDE,
                    GEOM_SPHERE, GEOM_CAPSULE, GEOM_BOX, GEOM_CYLINDER, GEOM_ELLIPSOID, DRIVE_POS,
                    DRIVE_EFFORT)

_GEOM_TYPES = {"sphere": GEOM_SPHERE, "capsule": GEOM_CAPSULE, "box": GEOM_BOX,
               "cylinder": GEOM_CYLINDER, "ellipsoid": GEOM_ELLIPSOID}


def _floats(s):
    return np.array([float(x) for x in s.split()], dtype=np.float64)


def _expand_includes(elem, base_dir):
    """Replace every <include file=.../> by the children of the included file's root, in place."""
    i = 0
    while i < len(elem):
        ch = elem[i]
        if ch.tag == "include":
            inc = ET.parse(os.path.join(base_dir, ch.attrib["file"])).getroot()
            _expand_includes(inc, base_dir)
            elem.remove(ch)
            for k, sub in enumerate(list(inc)):
                elem.insert(i + k, sub)
            i += len(list(inc))
        else:
            _expand_includes(ch, base_dir)
            i += 1


class _Defaults:
    """class name -> {tag -> attrib dict}, each class inheriting from its enclosing class."""

    def __init__(self, root):
        self.classes = {"main": {}}
        for d in root.findall("default"):
            self._walk(d, self.classes["main"])

    def _walk(self, d, parent_attrs):
        name = d.attrib.get("class", "main")
        cur = {k: dict(v) for k, v in parent_attrs.items()}
        for ch in d:
            if ch.tag != "default":
                cur.setdefault(ch.tag, {}).update(ch.attrib)
        self.classes[name] = cur
        for ch in d.findall("default"):
            self._walk(ch, cur)

    def resolve(self, elem, childclass):
        cls = elem.attrib.get("class", childclass or "main")
        out = dict(self.classes.get(cls, {}).get(elem.tag, {}))
        out.update(elem.attrib)
        return out


def load_mjcf(path, opts: BuildOptions = None, name=None):
    opts = opts or BuildOptions()
    tree = ET.parse(path)
    root = tree.getroot()
    _expand_includes(root, os.path.dirname(os.path.abspath(path)))
    comp = root.find("compiler")
    comp = comp.attrib if comp is not None else {}
    deg = comp.get("angle", "degree") == "degree"
    ang = np.pi / 180.0 if deg else 1.0
    defaults = _Defaults(root)

    def frame(a):
        pos = _floats(a["pos"]) if "pos" in a else np.zeros(3)
        if "quat" in a:
            R = rot.quat_to_mat(rot.quat_wxyz_to_xyzw(_floats(a["quat"])))
        elif "euler" in a:
            R = rot.euler_xyz_intrinsic_to_mat(_floats(a["euler"]) * ang)
        elif "axisangle" in a:
            v = _floats(a["axisangle"])
            R = rot.axis_angle_to_mat(v[:3], v[3] * ang)
        elif "zaxis" in a:
            R = rot.zaxis_to_mat(_floats(a["zaxis"]))
        else:
            R = np.eye(3)
        return pos, R

    state = {"free": False}

    def parse_body(be, childclass):
        childclass = be.attrib.get("childclass", childclass)
        pos, R = frame(be.attrib)
        b = IRBody(name=be.attrib.get("name", ""), pos=pos, R=R)
        for je in list(be.findall("freejoint")):
            state["free"] = True
        for je in be.findall("joint"):
            a = defaults.resolve(je, childclass)
            jt = a.get("type", "hinge")
            if jt == "free":
                state["free"] = True
                continue
            rng = _floats(a["range"]) if "range" in a else np.zeros(2)
            limited = a.get("limited", "auto")
            limited = ("range" in a) if limited == "auto" else (limited == "true")
            is_hinge = jt == "hinge"
            sc = ang if is_hinge else 1.0
            b.joints.append(IRJoint(
                name=a.get("name", ""), jtype=JOINT_HINGE if is_hinge else JOINT_SLIDE,
                axis=_floats(a.get("axis", "0 0 1")), anchor=_floats(a.get("pos", "0 0 0")),
                lower=rng[0] * sc, upper=rng[1] * sc, limited=limited,
                armature=float(a.get("armature", 0)), damping=float(a.get("damping", 0)),
                stiffness=float(a.get("stiffness", 0)), friction=float(a.get("frictionloss", 0))))
        ie = be.find("inertial")
        if ie is not None:
            ipos, iR = frame(ie.attrib)
            if "diaginertia" in ie.attrib:
                I = iR @ np.diag(_floats(ie.attrib["diaginertia"])) @ iR.T
            else:
                f = _floats(ie.attrib["fullinertia"])  # xx yy zz xy xz yz
                I = iR @ rot.sym6_to_mat(f) @ iR.T
            b.inertial = (float(ie.attrib["mass"]), ipos, I)
        for ge in be.findall("geom"):
            a = defaults.resolve(ge, childclass)
            gt = a.get("type", "sphere")
            if gt not in _GEOM_TYPES:     # mesh / plane / hfield: no primitive -> skipped
                if gt == "mesh" and int(a.get("contype", 1)) | int(a.get("conaffinity", 1)):       # a COLLIDING mesh: recorded, announced by build_model
                    b.skipped_geoms.append(a.get("name", a.get("mesh", "mesh")))
                continue
            size = _floats(a["size"]) if "size" in a else np.zeros(1)
            gpos, gR = frame(a)
            gtype = _GEOM_TYPES[gt]
            if "fromto" in a:
                ft = _floats(a["fromto"])
                p0, p1 = ft[:3], ft[3:]
                gpos = 0.5 * (p0 + p1)
                gR = rot.zaxis_to_mat(p1 - p0)
                size = np.array([size[0], 0.5 * np.linalg.norm(p1 - p0)])
            contype, conaff = int(a.get("contype", 1)), int(a.get("conaffinity", 1))
            b.geoms.append(IRGeom(
                name=a.get("name", ""), gtype=gtype, pos=gpos, R=gR, size=size,
                density=float(a.get("density", 1000.0)), mass=float(a.get("mass", -1.0)),
                friction=_floats(a.get("friction", "1 0.005 0.0001"))[0],
                collide=(contype != 0 or conaff != 0)))
        for se in be.findall("site"):
            a = defaults.resolve(se, childclass)
            b.sites[a.get("name", "")] = _floats(a.get("pos", "0 0 0"))
        for ce in be.findall("body"):
            b.children.append(parse_body(ce, childclass))
        return b

    wb = root.find("worldbody")
    top = wb.findall("body")
    if len(top) != 1:
        raise ValueError(f"{path}: expected exactly one top-level body, got {len(top)}")
    irroot = parse_body(top[0], None)
    model = build_model(name or root.attrib.get("model", os.path.basename(path)), irroot,
                        state["free"], opts)

    # actuators, in file order = the order the reference reads motor_effort in
    # (`ant.py:155-157`, `humanoid.py:160-161`)
    names, joints, kinds, gear, kp, fr = [], [], [], [], [], []
    act = root.find("actuator")
    if act is not None:
        for ae in act:
            if ae.tag not in ("motor", "position", "general"):
                continue
            a = defaults.resolve(ae, None)
            if a["joint"] not in model.dof_names:      # an included file's actuator for a joint this file has no body for (pen.xml includes the hand's shared.xml)
                continue
            names.append(a.get("name", a.get("joint", "")))
            joints.append(a["joint"]); kinds.append(ae.tag)
            gear.append(_floats(a.get("gear", "1"))[0])
            kp.append(float(a.get("kp", 0.0)))
            fr.append(_floats(a["forcerange"]) if "forcerange" in a else np.array([-1e30, 1e30]))
    model.actuator_names, model.actuator_joint, model.actuator_kind = names, joints, kinds
    model.actuator_gear = np.array(gear, dtype=np.float64)
    model.actuator_kp = np.array(kp, dtype=np.float64)
    model.actuator_forcerange = np.array(fr, dtype=np.float64).reshape(-1, 2)
    for k, jn in enumerate(joints):
        li = model.dof_names.index(jn) + 1
        if kinds[k] == "position":
            model.drive_mode[li] = DRIVE_POS
            model.kp[li] = kp[k]
            model.effort[li] = min(model.effort[li], abs(fr[k][1]))
        else:
            model.drive_mode[li] = DRIVE_EFFORT
    ten = root.find("tendon")
    if ten is not None:
        for fe in ten.findall("fixed"):
            if any(j.attrib["joint"] not in model.dof_names for j in fe.findall("joint")):
                continue
            rng = _floats(fe.attrib.get("range", "0 0"))
            model.tendons.append({
                "name": fe.attrib.get("name", ""),
                "dofs": [model.dof_names.index(j.attrib["joint"]) for j in fe.findall("joint")],
                "coefs": [float(j.attrib["coef"]) for j in fe.findall("joint")],
                "range": [float(rng[0]), float(rng[1])],
                "limited": fe.attrib.get("limited", "false") == "true",
                "limit_stiffness": 0.0, "damping": 0.0})
    finalize_limits(model)
    return model
