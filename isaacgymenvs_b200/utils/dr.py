"""Domain randomisation of the reference (`tasks/base/vec_task.py:610-840`, `utils/dr_utils.py:71-208`).

* observations / actions: the two "non-physical" entries of `task.randomization_params` -- noise lambdas on device tensors.
* actor_params: PHYSICAL properties.  The reference rewrites them actor by actor through `gym.set_actor_*_properties` in
  a Python loop over the envs being reset (vec_task.py:752-828); here they are per-env PARAMETER ARRAYS the step kernel
  reads (include/b200gym.h B2G_T_ENV_MASS_SCALE / ENV_DOF_PROPS / ENV_FRICTION), refreshed on the device for the envs
  that are about to reset and whose randomisation counter passed `frequency` -- the reference's selection rule
  (vec_task.py:631-637).  Supported: rigid_body_properties.mass, dof_properties.{damping, stiffness, lower, upper},
  rigid_shape_properties.{friction, restitution (scaled, no effect)}, sim_params.gravity (B2G_T_GRAVITY) for the tasks whose
  kernels read it (ShadowHand, Humanoid), and for a sim with a free object (ShadowHand: actors `hand` and `object`)
  tendon_properties and the object's scale, mass and friction (B2G_T_ENV_OBJ_PROPS / ENV_TENDON_DAMPING); anything else
  raises.

A NoiseModel is built from one YAML entry

    observations: {range: [0, .002], range_correlated: [0, .001], operation: additive, distribution: gaussian,
                   schedule: linear, schedule_steps: 40000}

and the simulation frame count (the schedule ramps the noise in).  Calling it perturbs a tensor with a per-step white
part and a correlated part whose unit sample is drawn once, the first time, and kept (`params['corr']` in the reference),
drawing from torch's global generator in the reference's order, so seeded runs reproduce the reference's numbers.
"""
import operator

import torch


def _schedule(entry, frame):
    kind = entry.get("schedule")
    if kind == "linear":
        return min(frame, entry["schedule_steps"]) / entry["schedule_steps"]
    if kind == "constant":
        return 0 if frame < entry["schedule_steps"] else 1
    return 1


class NoiseModel:
    def __init__(self, entry, frame, carry=None):
        self.dist = entry["distribution"]
        if self.dist not in ("gaussian", "uniform"):
            raise ValueError(f"unsupported noise distribution {self.dist!r} (gaussian | uniform)")
        self.additive = entry["operation"] == "additive"
        self.op = operator.add if self.additive else operator.mul
        a, b = entry["range"]
        ac, bc = entry.get("range_correlated", [0., 0.])
        s = _schedule(entry, frame)
        blend = (lambda v: v * s) if self.additive else (lambda v: v * s + 1.0 * (1.0 - s))
        if self.dist == "gaussian":                  # (mean, spread): under "scaling" only the mean is blended towards 1
            self.white = (blend(a), b * s)
            self.corr = (blend(ac), bc * s)
        else:                                        # (low, high): both ends blended
            self.white = (blend(a), blend(b))
            self.corr = (blend(ac), blend(bc))
        self.unit_corr = carry                       # the correlated part's unit sample survives re-parameterisation? no: the
        #                                              reference rebuilds its dict, dropping 'corr' -- carry stays None there

    def __call__(self, tensor):
        if self.unit_corr is None:
            self.unit_corr = torch.randn_like(tensor)
        if self.dist == "gaussian":
            mu, var = self.white
            mu_c, var_c = self.corr
            corr = self.unit_corr * var_c + mu_c
            return self.op(tensor, corr + torch.randn_like(tensor) * var + mu)
        lo, hi = self.white
        lo_c, hi_c = self.corr
        corr = self.unit_corr * (hi_c - lo_c) + lo_c
        return self.op(tensor, corr + torch.rand_like(tensor) * (hi - lo) + lo)


class Randomizer:
    """Frequency gating of `apply_randomizations` (vec_task.py:619-640) for the non-physical parameters: the noise models and,
    where the task's kernels read a bound gravity vector (`gravity` given: the sim's configured gravity), sim_params.gravity --
    the configured value plus a fresh sample per component each time the frequency elapsed (dr_utils.py:160-172)."""

    def __init__(self, dr_params, gravity=None, device=None):
        keys = ("frequency", "observations", "actions", "actor_params") + (("sim_params",) if gravity is not None else ())
        bad = [k for k in dr_params if k not in keys]
        if bad:
            raise NotImplementedError(f"domain randomisation of {bad} is not provided ({', '.join(keys[1:])})")
        bad = [k for k in dr_params.get("sim_params", {}) if k != "gravity"]
        if bad:
            raise NotImplementedError(f"sim_params {bad}: gravity only")
        self.params = dr_params
        self.freq = dr_params.get("frequency", 1)
        self.first = True
        self.last_rand_frame = 0
        self.models = {}
        self.og_gravity = self.gravity = None
        if "gravity" in dr_params.get("sim_params", {}):
            self.og_gravity = torch.tensor(gravity, dtype=torch.float32, device=device)
            self.gravity = self.og_gravity.clone()             # bound to the engine (B2G_T_GRAVITY), updated in place

    def update(self, frame):
        """Call before a step with the simulation frame count; re-parameterises the noise when the frequency elapsed."""
        due = self.first or (frame - self.last_rand_frame) >= self.freq
        if due:
            self.last_rand_frame = frame
            for key in ("observations", "actions"):
                if key in self.params:
                    self.models[key] = NoiseModel(self.params[key], frame)
            if self.gravity is not None:
                entry = self.params["sim_params"]["gravity"]
                smp = _sample(entry, (3,), frame, self.gravity.device)
                self.gravity.copy_(self.og_gravity * smp if entry["operation"] == "scaling" else self.og_gravity + smp)
        self.first = False
        return due


def _sched(entry, frame):
    return _schedule(entry, frame)


def _sample(entry, shape, frame, device, gen=None):
    """generate_random_samples, utils/dr_utils.py:71-131 (torch on the device instead of numpy on the host)."""
    a, b = entry["range"]
    s = _sched(entry, frame)
    additive = entry["operation"] == "additive"
    blend = (lambda v: v * s) if additive else (lambda v: v * s + 1.0 * (1.0 - s))
    dist = entry["distribution"]
    if dist == "gaussian":
        mu, var = blend(a), b * s
        return torch.randn(shape, device=device, generator=gen) * var + mu
    lo, hi = blend(a), blend(b)
    if dist == "loguniform":
        import math
        return torch.exp(torch.rand(shape, device=device, generator=gen) * (math.log(hi) - math.log(lo)) + math.log(lo))
    if dist == "uniform":
        return torch.rand(shape, device=device, generator=gen) * (hi - lo) + lo
    raise ValueError(f"unsupported distribution {dist!r}")


def _bucketed(val, entry):
    """get_bucketed_val, utils/dr_utils.py:135-145: the value rounded down onto `num_buckets` points spread over the sample
    range (uniform) or mean +- 2 sqrt(spread) (gaussian).  The reference's bisect wraps a value below the first point to the
    last point; here it is clamped to the first."""
    a, b = entry["range"]
    lo, hi = (a, b) if entry["distribution"] == "uniform" else (a - 2 * b ** 0.5, a + 2 * b ** 0.5)
    nb = int(entry["num_buckets"])
    k = torch.clamp(torch.floor((val - lo) / ((hi - lo) / nb)), 0, nb - 1)
    return (hi - lo) * k / nb + lo


class PhysicalRandomizer:
    """`actor_params` as per-env parameter tensors (see the module docstring), one entry per actor name.  `actors` maps each
    name to "articulation" or "object" (the free object of a ShadowHand-style sim); without it there must be exactly one
    actor type, the articulation.

    articulation: rigid_body_properties.mass, dof_properties.{damping, stiffness, lower, upper} (a position-driven DOF's damping
    is all of its velocity damping and its stiffness the drive's kp, as get_actor_dof_properties reports them),
    rigid_shape_properties.{friction, restitution}, and with tendons tendon_properties.{damping, stiffness}: the damping of
    each tendon; the active tendons' spring stiffness is 0 in the reference (shadow_hand.py:255-266), so scaling it changes
    nothing and it is drawn but not applied.  Restitution likewise: the MJCF shapes carry none (0), so under `scaling` it stays
    0 and is drawn but not applied (the contact model has no restitution); `additive` raises, as it would give the shapes a
    restitution the kernels do not model.
    object: scale (contact extents x s, inertia x s^2, mass unchanged: a modelling choice), rigid_body_properties.mass (mass,
    inertia and contact gains), rigid_shape_properties.friction.
    Friction is one value per env and actor (the reference draws one per shape); `num_buckets` rounds it onto the bucket grid."""
    SUPPORTED = {"rigid_body_properties": ("mass",), "dof_properties": ("damping", "stiffness", "lower", "upper"),
                 "rigid_shape_properties": ("friction", "restitution")}
    OBJECT_SUPPORTED = {"rigid_body_properties": ("mass",), "rigid_shape_properties": ("friction",)}

    def __init__(self, actor_params, model, num_envs, device, frequency, actors=None, obj=None, tendon_damping=None):
        self.bucketed = actors is not None                # num_buckets honoured for the multi-actor (ShadowHand) configs
        if actors is None:
            if len(actor_params) != 1:
                raise NotImplementedError("actor_params: exactly one actor type per environment")
            actors = {next(iter(actor_params)): "articulation"}
        self.entries = []                                  # (name, role, {group: {attr: entry}}), in the config's order
        for name, props in actor_params.items():
            role = actors.get(name)
            if role is None:
                raise NotImplementedError(f"actor_params.{name}: no such actor (actors: {sorted(actors)})")
            supported = dict(self.SUPPORTED) if role == "articulation" else dict(self.OBJECT_SUPPORTED)
            if role == "articulation" and tendon_damping is not None:
                supported["tendon_properties"] = ("damping", "stiffness")
            props = {k: v for k, v in props.items() if k != "color" and not (k == "scale" and role == "articulation")}
            for group, attrs in props.items():
                if group == "scale" and role == "object":
                    continue
                if group not in supported:
                    raise NotImplementedError(f"actor_params.{name}.{group} is not provided")
                for attr in attrs:
                    if attr not in supported[group]:
                        raise NotImplementedError(f"actor_params.{name}.{group}.{attr} is not provided")
                    if attr == "restitution" and attrs[attr]["operation"] != "scaling":
                        raise NotImplementedError(f"actor_params.{name}.{group}.restitution: scaling only (the shapes' restitution "
                                                  "is 0 and the contact model has none)")
            self.entries.append((name, role, props))
        art = [p for _, r, p in self.entries if r == "articulation"]
        ob = [p for _, r, p in self.entries if r == "object"]
        if len(art) > 1 or len(ob) > 1:
            raise NotImplementedError("actor_params: one articulation and at most one free object")
        if ob and obj is None:
            raise NotImplementedError("actor_params: an object entry needs a sim with a free object")
        self.props = art[0] if art else {}
        self.obj_props = ob[0] if ob else {}
        self.freq, self.N, self.device, self.first = frequency, num_envs, device, True
        f = lambda a: torch.tensor(a, dtype=torch.float32, device=device)
        nl, nd = model.nl, model.ndof
        import numpy as np
        lim = np.asarray(model.limited[1:]) > 0
        # a position-driven DOF (include/b200gym.h B2G_T_ENV_DOF_PROPS): damping = joint damping + the drive's kd, stiffness = kp
        pos = np.asarray(model.drive_mode[1:]) == 1
        damp = np.where(pos, np.asarray(model.damping[1:]) + np.asarray(model.kd[1:]), model.damping[1:]) if pos.any() else model.damping[1:]
        stiff = np.where(pos, model.kp[1:], model.stiffness[1:]) if pos.any() else model.stiffness[1:]
        self.og_dof = torch.stack([f(damp), f(stiff), f(np.where(lim, model.lower[1:], -3e38)),
                                   f(np.where(lim, model.upper[1:], 3e38))], -1)            # (nd, 4)
        self.limited = torch.tensor(lim, device=device)
        self.og_friction = float(np.asarray(model.cp_mu)[0]) if len(model.cp_mu) else 1.0
        self.mass_scale = torch.ones(num_envs, nl, device=device)
        self.dof_props = self.og_dof.unsqueeze(0).repeat(num_envs, 1, 1).contiguous()
        self.friction = torch.full((num_envs,), self.og_friction, device=device)
        self.uses = {g: g in self.props for g in self.SUPPORTED}
        self.uses["tendon_properties"] = "tendon_properties" in self.props
        self.og_tendon_damping = f(tendon_damping) if tendon_damping is not None else None
        self.tendon_damping = (self.og_tendon_damping.unsqueeze(0).repeat(num_envs, 1).contiguous()
                               if tendon_damping is not None else None)
        # the object: (size scale, mass factor, friction, unused) per env
        self.og_obj_friction = float(obj.get("mu", 1.0)) if obj is not None else 1.0
        self.obj_props_t = f([1.0, 1.0, self.og_obj_friction, 0.0]).unsqueeze(0).repeat(num_envs, 1).contiguous()

    def tensors(self, E):
        """slot -> tensor for the groups that are randomised."""
        out = {}
        if self.uses["rigid_body_properties"]:
            out[E.T_ENV_MASS_SCALE] = self.mass_scale
        if self.uses["dof_properties"]:
            out[E.T_ENV_DOF_PROPS] = self.dof_props
        if self.uses["rigid_shape_properties"]:
            out[E.T_ENV_FRICTION] = self.friction
        if self.uses["tendon_properties"]:
            out[E.T_ENV_TENDON_DAMPING] = self.tendon_damping
        if self.obj_props:
            out[E.T_ENV_OBJ_PROPS] = self.obj_props_t
        return out

    @torch.no_grad()
    def apply(self, frame, randomize_buf, reset_buf):
        """Re-sample the parameters of the envs selected by the reference's rule: all on the first call, afterwards the
        envs flagged for reset whose counter reached `frequency` (their counter restarts)."""
        if self.first:
            mask = torch.ones(self.N, dtype=torch.bool, device=self.device)
        else:
            mask = (randomize_buf >= self.freq) & (reset_buf != 0)
            randomize_buf[mask] = 0
        for _, role, props in self.entries:
            for group, attrs in props.items():
                if role == "object" and group == "scale":
                    self._draw_object(group, None, attrs, frame, mask)
                    continue
                for attr, entry in attrs.items():
                    if entry.get("setup_only", False) and not self.first:
                        continue
                    if role == "object":
                        self._draw_object(group, attr, entry, frame, mask)
                    else:
                        self._draw_articulation(group, attr, entry, frame, mask)
        self.first = False

    def _draw_articulation(self, group, attr, entry, frame, mask):
        N = self.N
        scaling = entry["operation"] == "scaling"
        if group == "rigid_body_properties":                       # mass, per body: here per link
            smp = _sample(entry, self.mass_scale.shape, frame, self.device)
            if not scaling:
                raise NotImplementedError("rigid_body_properties.mass: scaling only (the kernels take a factor)")
            self.mass_scale.copy_(torch.where(mask[:, None], smp, self.mass_scale))
        elif group == "dof_properties":
            col = ("damping", "stiffness", "lower", "upper").index(attr)
            og = self.og_dof[:, col]
            smp = _sample(entry, (N, og.shape[0]), frame, self.device)
            new = og[None] * smp if scaling else og[None] + smp
            if col >= 2:
                new = torch.where(self.limited[None], new, og[None])  # unlimited joints stay unlimited
            self.dof_props[:, :, col].copy_(torch.where(mask[:, None], new, self.dof_props[:, :, col]))
        elif group == "tendon_properties":                           # per tendon
            og = self.og_tendon_damping
            smp = _sample(entry, (N, og.shape[0]), frame, self.device)
            if attr == "damping":
                new = og[None] * smp if scaling else og[None] + smp
                self.tendon_damping.copy_(torch.where(mask[:, None], new, self.tendon_damping))
        elif attr == "restitution":                                  # a scaled 0: drawn, nothing to apply
            _sample(entry, (N,), frame, self.device)
        else:                                                        # friction: one value per env (all its shapes)
            smp = _sample(entry, (N,), frame, self.device)
            new = self.og_friction * smp if scaling else self.og_friction + smp
            if entry.get("num_buckets", 0) > 0 and self.bucketed:
                new = _bucketed(new, entry)
            self.friction.copy_(torch.where(mask, new, self.friction))

    def _draw_object(self, group, attr, entry, frame, mask):
        N = self.N
        if group == "scale":
            if entry.get("setup_only", False) and not self.first:
                return
            col, og = 0, 1.0
        elif group == "rigid_body_properties":
            col, og = 1, 1.0
            if entry["operation"] != "scaling":
                raise NotImplementedError("rigid_body_properties.mass: scaling only (the kernels take a factor)")
        else:
            col, og = 2, self.og_obj_friction
        smp = _sample(entry, (N,), frame, self.device)
        new = og * smp if entry["operation"] == "scaling" else og + smp
        if group == "rigid_shape_properties" and entry.get("num_buckets", 0) > 0:
            new = _bucketed(new, entry)
        self.obj_props_t[:, col].copy_(torch.where(mask, new, self.obj_props_t[:, col]))
