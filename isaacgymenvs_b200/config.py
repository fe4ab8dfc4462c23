"""Configuration for `make()`.

The reference composes hydra/OmegaConf YAML (`isaacgymenvs/__init__.py:29-41`, `cfg/config.yaml`,
`cfg/task/*.yaml`); hydra and omegaconf are not part of this image, so this module has
  * `load_reference_cfg(cfg_dir, task, overrides)`: a small YAML + interpolation loader that reads an
    UNMODIFIED reference-format config tree (relative `${..x}` references, the four resolvers
    registered at `isaacgymenvs/__init__.py:8-11`), and
  * `builtin_cfg(task, overrides)`: the same dictionaries for the supported tasks, written out as
    Python so the package works where no reference tree exists (the GPU box).
Both return plain nested dicts shaped like `omegaconf_to_dict(cfg.task)` plus the root keys.
"""
import copy
import os
import re

ROOT_DEFAULTS = {   # cfg/config.yaml:1-59
    "task_name": None, "experiment": "", "num_envs": "", "seed": 42, "torch_deterministic": False,
    "max_iterations": "", "physics_engine": "physx", "pipeline": "gpu", "sim_device": "cuda:0",
    "rl_device": "cuda:0", "graphics_device_id": 0, "num_threads": 4, "solver_type": 1, "num_subscenes": 4,
    "test": False, "checkpoint": "", "sigma": "", "multi_gpu": False, "capture_video": False,
    "force_render": True, "headless": False,
}


def _physx(root, **kw):
    d = {"num_threads": root["num_threads"], "solver_type": root["solver_type"],
         "use_gpu": "cuda" in str(root["sim_device"]), "num_position_iterations": 4, "num_velocity_iterations": 0,
         "contact_offset": 0.02, "rest_offset": 0.0, "bounce_threshold_velocity": 0.2,
         "max_depenetration_velocity": 10.0, "default_buffer_size_multiplier": 5.0,
         "max_gpu_contact_pairs": 8388608, "num_subscenes": root["num_subscenes"], "contact_collection": 0}
    d.update(kw)
    return d


def _sim(root, physx):
    return {"dt": 0.0166, "substeps": 2, "up_axis": "z", "use_gpu_pipeline": root["pipeline"] == "gpu",
            "gravity": [0.0, 0.0, -9.81], "physx": physx}


def _num_envs(root, default):
    return default if root["num_envs"] in ("", None) else int(root["num_envs"])


# the reference's randomization_params blocks: what task.randomize=True turns on
def _dr(lo, hi, op, dist, **kw):
    return {"range": [lo, hi], "operation": op, "distribution": dist, **kw}


# cfg/task/ShadowHand.yaml (the same block as ShadowHandOpenAI_FF.yaml / ShadowHandTest.yaml)
_SHADOW_HAND_DR = {
    "frequency": 720,
    "observations": _dr(0, .002, "additive", "gaussian", range_correlated=[0, .001]),
    "actions": _dr(0., .05, "additive", "gaussian", range_correlated=[0, .015]),
    "sim_params": {"gravity": _dr(0, 0.4, "additive", "gaussian")},
    "actor_params": {
        "hand": {"color": True,
                 "tendon_properties": {"damping": _dr(0.3, 3.0, "scaling", "loguniform"),
                                       "stiffness": _dr(0.75, 1.5, "scaling", "loguniform")},
                 "dof_properties": {"damping": _dr(0.3, 3.0, "scaling", "loguniform"),
                                    "stiffness": _dr(0.75, 1.5, "scaling", "loguniform"),
                                    "lower": _dr(0, 0.01, "additive", "gaussian"), "upper": _dr(0, 0.01, "additive", "gaussian")},
                 "rigid_body_properties": {"mass": _dr(0.5, 1.5, "scaling", "uniform", setup_only=True)},
                 "rigid_shape_properties": {"friction": _dr(0.7, 1.3, "scaling", "uniform", num_buckets=250)}},
        "object": {"scale": _dr(0.95, 1.05, "scaling", "uniform", setup_only=True),
                   "rigid_body_properties": {"mass": _dr(0.5, 1.5, "scaling", "uniform", setup_only=True)},
                   "rigid_shape_properties": {"friction": _dr(0.7, 1.3, "scaling", "uniform", num_buckets=250)}}}}


# cfg/task/Ant.yaml and cfg/task/Humanoid.yaml randomization_params
_ANT_DR = {
    "frequency": 600,
    "observations": _dr(0, .002, "additive", "gaussian"),
    "actions": _dr(0., .02, "additive", "gaussian"),
    "actor_params": {
        "ant": {"color": True,
                "rigid_body_properties": {"mass": _dr(0.5, 1.5, "scaling", "uniform", setup_only=True)},
                "dof_properties": {"damping": _dr(0.5, 1.5, "scaling", "uniform"), "stiffness": _dr(0.5, 1.5, "scaling", "uniform"),
                                   "lower": _dr(0, 0.01, "additive", "gaussian"), "upper": _dr(0, 0.01, "additive", "gaussian")}}}}


def _lin(lo, hi, op, dist, **kw):          # Humanoid.yaml's entries ramp in over 3000 frames
    return _dr(lo, hi, op, dist, **kw, schedule="linear", schedule_steps=3000)


_HUMANOID_DR = {
    "frequency": 600,
    "observations": _dr(0, .002, "additive", "gaussian"),
    "actions": _dr(0., .02, "additive", "gaussian"),
    "sim_params": {"gravity": _lin(0, 0.4, "additive", "gaussian")},
    "actor_params": {
        "humanoid": {"color": True,
                     "rigid_body_properties": {"mass": _lin(0.5, 1.5, "scaling", "uniform", setup_only=True)},
                     "rigid_shape_properties": {"friction": _lin(0.7, 1.3, "scaling", "uniform", num_buckets=500),
                                                "restitution": _lin(0., 0.7, "scaling", "uniform")},
                     "dof_properties": {"damping": _lin(0.5, 1.5, "scaling", "uniform"), "stiffness": _lin(0.5, 1.5, "scaling", "uniform"),
                                        "lower": _lin(0, 0.01, "additive", "gaussian"), "upper": _lin(0, 0.01, "additive", "gaussian")}}}}


def _builtin_task(name, root):
    """Python restatement of cfg/task/{Cartpole,Ant,Humanoid}.yaml (values only)."""
    plane = {"staticFriction": 1.0, "dynamicFriction": 1.0, "restitution": 0.0}
    if name == "Cartpole":
        return {"name": "Cartpole", "physics_engine": root["physics_engine"],
                "env": {"numEnvs": _num_envs(root, 512), "envSpacing": 4.0, "resetDist": 3.0, "maxEffort": 400.0,
                        "clipObservations": 5.0, "clipActions": 1.0,
                        "asset": {"assetRoot": "../../assets", "assetFileName": "urdf/cartpole.urdf"},
                        "enableCameraSensors": False},
                "sim": _sim(root, _physx(root, rest_offset=0.001, max_depenetration_velocity=100.0,
                                         default_buffer_size_multiplier=2.0, max_gpu_contact_pairs=1048576)),
                "task": {"randomize": False}}
    if name == "Ant":
        return {"name": "Ant", "physics_engine": root["physics_engine"],
                "env": {"numEnvs": _num_envs(root, 4096), "envSpacing": 5, "episodeLength": 1000,
                        "enableDebugVis": False, "clipActions": 1.0, "powerScale": 1.0, "controlFrequencyInv": 1,
                        "headingWeight": 0.5, "upWeight": 0.1, "actionsCost": 0.005, "energyCost": 0.05,
                        "dofVelocityScale": 0.2, "contactForceScale": 0.1, "jointsAtLimitCost": 0.1,
                        "deathCost": -2.0, "terminationHeight": 0.31, "plane": plane,
                        "asset": {"assetFileName": "mjcf/nv_ant.xml"}, "enableCameraSensors": False},
                "sim": _sim(root, _physx(root)),
                "task": {"randomize": False, "randomization_params": copy.deepcopy(_ANT_DR)}}
    if name == "Humanoid":
        return {"name": "Humanoid", "physics_engine": root["physics_engine"],
                "env": {"numEnvs": _num_envs(root, 4096), "envSpacing": 5, "episodeLength": 1000,
                        "enableDebugVis": False, "clipActions": 1.0, "powerScale": 1.0,
                        "headingWeight": 0.5, "upWeight": 0.1, "actionsCost": 0.01, "energyCost": 0.05,
                        "dofVelocityScale": 0.1, "angularVelocityScale": 0.25, "contactForceScale": 0.01,
                        "jointsAtLimitCost": 0.25, "deathCost": -1.0, "terminationHeight": 0.8, "plane": plane,
                        "asset": {"assetFileName": "mjcf/nv_humanoid.xml"}, "enableCameraSensors": False},
                "sim": _sim(root, _physx(root)),
                "task": {"randomize": False, "randomization_params": copy.deepcopy(_HUMANOID_DR)}}
    if name == "ShadowHand":
        sim = _sim(root, _physx(root, num_position_iterations=8, contact_offset=0.002, max_depenetration_velocity=1000.0))
        sim.update({"dt": 0.01667, "substeps": 2})
        return {"name": "ShadowHand", "physics_engine": root["physics_engine"],
                "env": {"numEnvs": _num_envs(root, 16384), "envSpacing": 0.75, "episodeLength": 600, "enableDebugVis": False,
                        "aggregateMode": 1, "clipObservations": 5.0, "clipActions": 1.0, "stiffnessScale": 1.0,
                        "forceLimitScale": 1.0, "useRelativeControl": False, "dofSpeedScale": 20.0,
                        "actionsMovingAverage": 1.0, "controlFrequencyInv": 1, "startPositionNoise": 0.01,
                        "startRotationNoise": 0.0, "resetPositionNoise": 0.01, "resetRotationNoise": 0.0,
                        "resetDofPosRandomInterval": 0.2, "resetDofVelRandomInterval": 0.0, "forceScale": 0.0,
                        "forceProbRange": [0.001, 0.1], "forceDecay": 0.99, "forceDecayInterval": 0.08,
                        "distRewardScale": -10.0, "rotRewardScale": 1.0, "rotEps": 0.1, "actionPenaltyScale": -0.0002,
                        "reachGoalBonus": 250, "fallDistance": 0.24, "fallPenalty": 0.0, "objectType": "block",
                        "observationType": "full_state", "asymmetric_observations": False, "successTolerance": 0.1,
                        "printNumSuccesses": False, "maxConsecutiveSuccesses": 0,
                        "asset": {"assetFileName": "mjcf/open_ai_assets/hand/shadow_hand.xml",
                                  "assetFileNameBlock": "urdf/objects/cube_multicolor.urdf",
                                  "assetFileNameEgg": "mjcf/open_ai_assets/hand/egg.xml",
                                  "assetFileNamePen": "mjcf/open_ai_assets/hand/pen.xml"},
                        "enableCameraSensors": False},
                "sim": sim,
                "task": {"randomize": False, "randomization_params": copy.deepcopy(_SHADOW_HAND_DR)}}
    if name == "AnymalTerrain":
        sim = _sim(root, _physx(root, num_velocity_iterations=1, max_depenetration_velocity=100.0, contact_collection=1))
        sim.update({"dt": 0.005, "substeps": 1})
        return {"name": "AnymalTerrain", "physics_engine": "physx",
                "env": {"numEnvs": _num_envs(root, 4096), "numObservations": 188, "numActions": 12, "envSpacing": 3.,
                        "enableDebugVis": False,
                        "terrain": {"terrainType": "trimesh", "staticFriction": 1.0, "dynamicFriction": 1.0, "restitution": 0.,
                                    "curriculum": True, "maxInitMapLevel": 0, "mapLength": 8., "mapWidth": 8., "numLevels": 10,
                                    "numTerrains": 20, "terrainProportions": [0.1, 0.1, 0.35, 0.25, 0.2], "slopeTreshold": 0.5},
                        "baseInitState": {"pos": [0.0, 0.0, 0.62], "rot": [0.0, 0.0, 0.0, 1.0], "vLinear": [0.0, 0.0, 0.0],
                                          "vAngular": [0.0, 0.0, 0.0]},
                        "randomCommandVelocityRanges": {"linear_x": [-1., 1.], "linear_y": [-1., 1.], "yaw": [-3.14, 3.14]},
                        "control": {"stiffness": 80.0, "damping": 2.0, "actionScale": 0.5, "decimation": 4},
                        "defaultJointAngles": {"LF_HAA": 0.03, "LH_HAA": 0.03, "RF_HAA": -0.03, "RH_HAA": -0.03,
                                               "LF_HFE": 0.4, "LH_HFE": -0.4, "RF_HFE": 0.4, "RH_HFE": -0.4,
                                               "LF_KFE": -0.8, "LH_KFE": 0.8, "RF_KFE": -0.8, "RH_KFE": 0.8},
                        "urdfAsset": {"file": "urdf/anymal_c/urdf/anymal_minimal.urdf", "footName": "SHANK", "kneeName": "THIGH",
                                      "collapseFixedJoints": True, "fixBaseLink": False, "defaultDofDriveMode": 4},
                        "learn": {"allowKneeContacts": True, "terminalReward": 0.0, "linearVelocityXYRewardScale": 1.0,
                                  "linearVelocityZRewardScale": -4.0, "angularVelocityXYRewardScale": -0.05,
                                  "angularVelocityZRewardScale": 0.5, "orientationRewardScale": -0., "torqueRewardScale": -0.00002,
                                  "jointAccRewardScale": -0.0005, "baseHeightRewardScale": -0.0, "feetAirTimeRewardScale": 1.0,
                                  "kneeCollisionRewardScale": -0.25, "feetStumbleRewardScale": -0., "actionRateRewardScale": -0.01,
                                  "hipRewardScale": -0., "linearVelocityScale": 2.0, "angularVelocityScale": 0.25,
                                  "dofPositionScale": 1.0, "dofVelocityScale": 0.05, "heightMeasurementScale": 5.0,
                                  "addNoise": True, "noiseLevel": 1.0, "dofPositionNoise": 0.01, "dofVelocityNoise": 1.5,
                                  "linearVelocityNoise": 0.1, "angularVelocityNoise": 0.2, "gravityNoise": 0.05,
                                  "heightMeasurementNoise": 0.06, "randomizeFriction": True, "frictionRange": [0.5, 1.25],
                                  "pushRobots": True, "pushInterval_s": 15, "episodeLength_s": 20},
                        "viewer": {"refEnv": 0, "pos": [0, 0, 10], "lookat": [1., 1, 9]}, "enableCameraSensors": False},
                "sim": sim, "task": {"randomize": False}}
    raise KeyError(f"no built-in config for task {name!r}; pass cfg_dir= pointing at a reference-format cfg tree")


def builtin_cfg(task, overrides=None):
    root = copy.deepcopy(ROOT_DEFAULTS)
    root.update(overrides or {})
    root["task_name"] = task
    root["task"] = _builtin_task(task, root)
    return root


# ------------------------------------------------------------------------- reference-format YAML
_INTERP = re.compile(r"\$\{([^${}]*)\}")


def _split_args(s):
    out, depth, cur, quote = [], 0, "", None
    for ch in s:
        if quote:
            cur += ch
            if ch == quote:
                quote = None
        elif ch in "\"'":
            quote = ch; cur += ch
        elif ch == "," and depth == 0:
            out.append(cur.strip()); cur = ""
        else:
            cur += ch
    out.append(cur.strip())
    return out


def _lit(s):
    if isinstance(s, str):
        t = s.strip()
        if len(t) >= 2 and t[0] == t[-1] and t[0] in "\"'":
            return t[1:-1]
        low = t.lower()
        if low in ("true", "false"):
            return low == "true"
        if low in ("null", "none"):
            return None
        try:
            return int(t)
        except ValueError:
            try:
                return float(t)
            except ValueError:
                return t
    return s


def _resolver(name, args):
    a = [_lit(x) for x in args]
    if name == "eq":            # isaacgymenvs/__init__.py:8
        return str(a[0]).lower() == str(a[1]).lower()
    if name == "contains":      # :9
        return str(a[0]).lower() in str(a[1]).lower()
    if name == "if":            # :10
        return a[1] if a[0] else a[2]
    if name == "resolve_default":   # :11
        return a[0] if a[1] in ("", None) else a[1]
    raise KeyError(f"unknown resolver {name}")


def _get_path(root, path, here):
    """OmegaConf reference: leading dots climb from the node's PARENT container."""
    if path.startswith("."):
        n = len(path) - len(path.lstrip("."))
        base = here[:len(here) - n] if n <= len(here) else []
        keys = base + [k for k in path.lstrip(".").split(".") if k]
    else:
        keys = path.split(".")
    node = root
    for k in keys:
        node = node[k]
    return node


def _resolve_str(root, s, here):
    while True:
        m = _INTERP.search(s)
        if not m:
            return _lit(s) if s != "" else s
        inner = m.group(1)
        if ":" in inner and not inner.startswith("."):
            name, rest = inner.split(":", 1)
            val = _resolver(name.strip(), _split_args(rest))
        else:
            val = _get_path(root, inner.strip(), here)
            if isinstance(val, str) and "${" in val:
                val = _resolve_str(root, val, here)
        if m.start() == 0 and m.end() == len(s):
            return val
        rep = f'"{val}"' if isinstance(val, str) and "," in val else str(val)
        s = s[:m.start()] + rep + s[m.end():]


def _resolve_tree(root, node, here):
    if isinstance(node, dict):
        for k in list(node.keys()):
            node[k] = _resolve_tree(root, node[k], here + [k])
        return node
    if isinstance(node, list):
        return [_resolve_tree(root, v, here + [str(i)]) for i, v in enumerate(node)]
    if isinstance(node, str) and "${" in node:
        return _resolve_str(root, node, here[:-1] + [here[-1]])
    return node


def load_reference_cfg(cfg_dir, task, overrides=None):
    """Compose `<cfg_dir>/config.yaml` + `<cfg_dir>/task/<task>.yaml` the way hydra would for
    `task=<task>` (cfg/config.yaml:60-66), minus the train/pbt groups the env never reads."""
    import yaml
    with open(os.path.join(cfg_dir, "config.yaml")) as f:
        root = yaml.safe_load(f)
    for k in ("defaults", "hydra"):
        root.pop(k, None)
    for k in list(root.keys()):   # keys that interpolate into the absent train group
        if isinstance(root[k], str) and "${train" in root[k]:
            root[k] = ""
    root.update(overrides or {})
    with open(os.path.join(cfg_dir, "task", f"{task}.yaml")) as f:
        root["task"] = yaml.safe_load(f)
    root["task_name"] = root["task"].get("name", task)
    return _resolve_tree(root, root, [])
