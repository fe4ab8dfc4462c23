#!/usr/bin/env python
"""tools/train_ppo.py -- a compact PPO learner driving the env through the reference's wrapper surface
(utils/rlgames_utils.py:242-295 RLGPUEnv: env.reset() / env.step(actions) with dict observations, `time_outs` in the
info dict for value bootstrap), with the hyper-parameters of the reference's cfg/train/AntPPO.yaml (a2c_continuous,
[256,128,64] ELU MLP, fixed sigma, lr 3e-4 with the adaptive-KL schedule, gamma 0.99, tau 0.95, horizon 16,
minibatch 32768, 4 mini-epochs, e_clip 0.2, critic_coef 2, normalised inputs / values / advantages, reward scale 0.01,
bounds loss 1e-4).  rl_games itself is not installable here (no network); this is the smallest learner that exercises
the same contract and answers the question the parity tests cannot: does Ant LEARN on this physics?

    python tools/train_ppo.py --task Ant --num-envs 4096 --epochs 500 --out ppo_ant.json
"""
import argparse
import json
import os
import sys
import time

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class RunningMeanStd(nn.Module):
    def __init__(self, shape, eps=1e-5):
        super().__init__()
        self.register_buffer("mean", torch.zeros(shape)); self.register_buffer("var", torch.ones(shape)); self.register_buffer("count", torch.ones(()))
        self.eps = eps

    @torch.no_grad()
    def update(self, x):
        x = x.reshape(-1, *self.mean.shape) if self.mean.dim() else x.reshape(-1)
        bm, bv, bc = x.mean(0), x.var(0, unbiased=False), x.shape[0]
        d = bm - self.mean
        tot = self.count + bc
        self.mean += d * bc / tot
        self.var.copy_((self.var * self.count + bv * bc + d * d * self.count * bc / tot) / tot)
        self.count.copy_(tot)

    def norm(self, x, clip=5.0):
        return torch.clamp((x - self.mean) / torch.sqrt(self.var + self.eps), -clip, clip)

    def denorm(self, y):
        return y * torch.sqrt(self.var + self.eps) + self.mean


class ActorCritic(nn.Module):
    def __init__(self, nobs, nact, units=(256, 128, 64)):
        super().__init__()
        layers, d = [], nobs
        for u in units:
            layers += [nn.Linear(d, u), nn.ELU()]
            d = u
        self.trunk = nn.Sequential(*layers)
        self.mu = nn.Linear(d, nact); self.value = nn.Linear(d, 1)
        self.logstd = nn.Parameter(torch.zeros(nact))          # fixed_sigma: a state-independent parameter, initialised to 0

    def forward(self, x):
        h = self.trunk(x)
        return self.mu(h), self.logstd.expand(x.shape[0], -1), self.value(h).squeeze(-1)


def neglogp(a, mu, logstd):
    return 0.5 * (((a - mu) / logstd.exp()) ** 2).sum(-1) + logstd.sum(-1) + 0.5 * a.shape[-1] * 1.8378770664093453


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--task", default="Ant")
    ap.add_argument("--num-envs", type=int, default=4096)
    ap.add_argument("--epochs", type=int, default=500)
    ap.add_argument("--horizon", type=int, default=16)
    ap.add_argument("--minibatch", type=int, default=32768)
    ap.add_argument("--seed", type=int, default=42)
    ap.add_argument("--out", default="")
    ap.add_argument("--device", default="cuda:0")
    ap.add_argument("--units", default="256,128,64")          # HumanoidPPO.yaml: 400,200,100
    ap.add_argument("--lr", type=float, default=3e-4)          # HumanoidPPO.yaml: 5e-4
    ap.add_argument("--mini-epochs", type=int, default=4)      # HumanoidPPO.yaml: 5
    ap.add_argument("--critic-coef", type=float, default=2.0)  # HumanoidPPO.yaml: 4
    ap.add_argument("--self-collision", action="store_true")   # Humanoid: env.selfCollision=True
    ap.add_argument("--kl-threshold", type=float, default=0.008)   # ShadowHandPPO.yaml: 0.016
    ap.add_argument("--reward-scale", type=float, default=0.01)    # reward_shaper.scale_value; CartpolePPO.yaml 0.1, AnymalTerrainPPO.yaml 1.0
    ap.add_argument("--bounds-coef", type=float, default=1e-4)     # bounds_loss_coef; AnymalTerrainPPO.yaml 0
    ap.add_argument("--env", default="", help="comma-separated overrides of cfg.task.env, e.g. objectType=pen,forceScale=2.0")
    args = ap.parse_args(argv)
    import isaacgymenvs_b200
    dev = args.device
    torch.manual_seed(args.seed)
    cfg = None
    if args.self_collision:
        from isaacgymenvs_b200 import config
        cfg = config.builtin_cfg(args.task, {"sim_device": dev, "rl_device": dev}); cfg["task"]["env"]["selfCollision"] = True
    if args.env:
        from isaacgymenvs_b200 import config
        cfg = cfg or config.builtin_cfg(args.task, {"sim_device": dev, "rl_device": dev})
        for kv in args.env.split(","):
            k, v = kv.split("=")
            try:
                v = float(v) if "." in v or "e" in v.lower() else int(v)
            except ValueError:
                pass
            cfg["task"]["env"][k] = v
    env = isaacgymenvs_b200.make(seed=args.seed, task=args.task, num_envs=args.num_envs, sim_device=dev, rl_device=dev, headless=True, cfg=cfg)
    N, O, A, T = env.num_envs, env.num_obs, env.num_acts, args.horizon
    net = ActorCritic(O, A, tuple(int(u) for u in args.units.split(","))).to(dev)
    obs_rms, val_rms = RunningMeanStd((O,)).to(dev), RunningMeanStd(()).to(dev)
    lr, kl_thr, gamma, tau, e_clip, critic_coef, bounds_coef, rew_scale = args.lr, args.kl_threshold, 0.99, 0.95, 0.2, args.critic_coef, args.bounds_coef, args.reward_scale
    opt = torch.optim.Adam(net.parameters(), lr=lr, eps=1e-8)
    obs = env.reset()["obs"].clone()
    ep_ret = torch.zeros(N, device=dev); ep_len = torch.zeros(N, device=dev)
    done_ret, done_len = [], []
    log = []
    B = N * T
    mb = min(args.minibatch, B)
    t_start = time.time()
    env_steps = 0
    for epoch in range(args.epochs):
        bo = torch.zeros(T, N, O, device=dev); ba = torch.zeros(T, N, A, device=dev); bnlp = torch.zeros(T, N, device=dev)
        bv = torch.zeros(T, N, device=dev); br = torch.zeros(T, N, device=dev); bd = torch.zeros(T, N, device=dev)
        bmu = torch.zeros(T, N, A, device=dev)
        with torch.no_grad():
            for t in range(T):
                obs_rms.update(obs)
                mu, logstd, v = net(obs_rms.norm(obs))
                a = mu + logstd.exp() * torch.randn_like(mu)
                bo[t], ba[t], bmu[t], bnlp[t], bv[t] = obs, a, mu, neglogp(a, mu, logstd), val_rms.denorm(v)
                od, rew, done, info = env.step(torch.clamp(a, -1.0, 1.0))
                obs = od["obs"].clone()
                r = rew.clone() * rew_scale
                # value_bootstrap: an episode that merely timed out keeps the value of the state it was cut at
                r = r + gamma * bv[t] * info["time_outs"].float()
                br[t], bd[t] = r, done.float()
                ep_ret += rew; ep_len += 1
                fin = done.nonzero(as_tuple=False).flatten()
                if len(fin):
                    done_ret.append(ep_ret[fin].clone()); done_len.append(ep_len[fin].clone())
                    ep_ret[fin] = 0; ep_len[fin] = 0
            env_steps += N * T
            _, _, v_last = net(obs_rms.norm(obs))
            v_last = val_rms.denorm(v_last)
            adv = torch.zeros(T, N, device=dev); last = torch.zeros(N, device=dev)
            for t in reversed(range(T)):
                nv = v_last if t == T - 1 else bv[t + 1]
                nonterm = 1.0 - bd[t]
                delta = br[t] + gamma * nv * nonterm - bv[t]
                last = delta + gamma * tau * nonterm * last
                adv[t] = last
            ret = adv + bv
            val_rms.update(ret); val_rms.update(bv)
            f = lambda x: x.reshape(B, *x.shape[2:])
            fo, fa, fnlp, fadv, fret, fv, fmu = f(bo), f(ba), f(bnlp), f(adv), val_rms.norm(f(ret), clip=1e9), val_rms.norm(f(bv), clip=1e9), f(bmu)
            fadv = (fadv - fadv.mean()) / (fadv.std() + 1e-8)
            fon = obs_rms.norm(fo)
        kls = []
        for _ in range(args.mini_epochs):
            perm = torch.randperm(B, device=dev)
            for s in range(0, B, mb):
                idx = perm[s:s + mb]
                mu, logstd, v = net(fon[idx])
                nlp = neglogp(fa[idx], mu, logstd)
                ratio = torch.exp(fnlp[idx] - nlp)
                a_loss = torch.max(-fadv[idx] * ratio, -fadv[idx] * torch.clamp(ratio, 1 - e_clip, 1 + e_clip)).mean()
                v_clip = fv[idx] + torch.clamp(v - fv[idx], -e_clip, e_clip)
                c_loss = torch.max((v - fret[idx]) ** 2, (v_clip - fret[idx]) ** 2).mean()
                b_loss = (torch.clamp(mu - 1.1, min=0) ** 2 + torch.clamp(-1.1 - mu, min=0) ** 2).sum(-1).mean()
                loss = a_loss + 0.5 * critic_coef * c_loss + bounds_coef * b_loss
                opt.zero_grad(set_to_none=True)
                loss.backward()
                nn.utils.clip_grad_norm_(net.parameters(), 1.0)
                opt.step()
                with torch.no_grad():      # KL(old || new) of the diagonal Gaussians, for the adaptive schedule
                    kl = (((fmu[idx] - mu) ** 2) / (2 * (2 * logstd).exp())).sum(-1)      # sigma moves slowly: the mean term
                    kls.append(kl.mean())
        kl = torch.stack(kls).mean().item()
        if kl > 2.0 * kl_thr:
            lr = max(lr / 1.5, 1e-6)
        if kl < 0.5 * kl_thr:
            lr = min(lr * 1.5, 1e-2)
        for g in opt.param_groups:
            g["lr"] = lr
        if done_ret:
            dr = torch.cat(done_ret); dl = torch.cat(done_len)
            mean_ret, mean_len, nfin = dr.mean().item(), dl.mean().item(), int(dr.numel())
            done_ret, done_len = [], []
        else:
            mean_ret, mean_len, nfin = float("nan"), float("nan"), 0
        rec = dict(epoch=epoch, env_steps=env_steps, mean_episode_return=mean_ret, mean_episode_length=mean_len, episodes=nfin,
                   mean_step_reward=float(br.mean().item() / rew_scale), kl=kl, lr=lr, wall_s=time.time() - t_start)
        log.append(rec)
        if epoch % 10 == 0 or epoch == args.epochs - 1:
            print(json.dumps(rec), flush=True)
    if dev.startswith("cuda"):
        torch.cuda.synchronize()
    wall = time.time() - t_start
    first = [r["mean_step_reward"] for r in log[:10]]; lastr = [r["mean_step_reward"] for r in log[-10:]]
    summary = dict(task=args.task, num_envs=N, epochs=args.epochs, env_steps=env_steps, wall_s=wall, env_steps_per_s_incl_learner=env_steps / wall,
                   mean_step_reward_first10=sum(first) / len(first), mean_step_reward_last10=sum(lastr) / len(lastr),
                   best_mean_episode_return=max((r["mean_episode_return"] for r in log if r["episodes"] > 0), default=float("nan")),
                   hyperparameters=f"a2c_continuous as cfg/train/{args.task}PPO.yaml: units {args.units}, lr {args.lr} adaptive kl 0.008, gamma 0.99, tau 0.95, horizon {args.horizon}, minibatch {args.minibatch}, {args.mini_epochs} mini-epochs, e_clip 0.2, critic_coef {args.critic_coef}",
                   self_collision=bool(args.self_collision))
    print(json.dumps(summary), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(dict(summary=summary, curve=log[:: max(1, len(log) // 100)]), fh, indent=1)


if __name__ == "__main__":
    main()
