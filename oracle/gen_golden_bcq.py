"""TEST INFRASTRUCTURE -- golden vectors for BCQ from the UNMODIFIED reference (thu-ml/tianshou 2.0.1 imported through
oracle/ref_shim.py), run on the CPU.

    python -m oracle.gen_golden_bcq       # writes tests/golden/bcq_ref_{d4rl,net,small}.npz

Cases:
  d4rl  : the examples/offline/d4rl_bcq.py shape -- obs 17, act 6, an MLP perturbation of [256, 256] (row 0 perturbs the whole
          batch), Net critics of [256, 256], a VAE of [512, 512] with latent 12, batch 256, N = 10, a ``from_data`` buffer;
          compact: parameters after the last update only, each as ``golden_view``
  net   : a Net perturbation (every row its own), a separate critic2 with its own optimiser, max_action = 2 and phi = 3 (the
          +-max_action clamp binds), lmbda = 0.5, N = 1, a buffer where many rows are done
  small : the test/offline/test_bcq.py shape (obs 3, act 1, max_action 2, hidden [64], VAE [32, 32]), plus the actions
          BCQPolicy.forward picks for 10 observations after the updates and torch's CPU generator state after that
Every network's initial weights come from ``oracle_discrete_sac.seeded_params`` (the seed is stored, not the tensors).  Captured:
the buffer, the reference's state_dict() keys, and per ``update()`` the sampled indices, the four losses, the torch CPU generator
state and the parameters of the perturbation network, both critics, the VAE and the three lagged networks.  Before update u the
recipe seeds numpy with 500 + u and torch with 100 + u; before the policy call torch with 900.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "tests", "golden")

from oracle.oracle_discrete_sac import golden_view, seeded_params  # noqa: E402
from oracle.ref_shim import import_reference  # noqa: E402

ts = import_reference()
from gymnasium.spaces import Box  # noqa: E402  (shim stand-in)
from tianshou.algorithm.imitation.bcq import BCQ, BCQPolicy  # noqa: E402
from tianshou.algorithm.optim import AdamOptimizerFactory  # noqa: E402
from tianshou.data import Batch, ReplayBuffer  # noqa: E402
from tianshou.utils.net.common import MLP, Net  # noqa: E402
from tianshou.utils.net.continuous import VAE, ContinuousCritic, Perturbation  # noqa: E402
from tianshou.utils.torch_utils import policy_within_training_step  # noqa: E402

_BASE = dict(gamma=0.99, tau=0.005, lmbda=0.75, N=10, phi=0.05, max_action=1.0, per_row=False, critic2=False, actor_lr=1e-3,
             critic_lr=1e-3, critic2_lr=1e-3, vae_lr=1e-3, p_done=0.05, S=100, policy_obs=0, compact=False, init_seed=40)
VARIANTS = {
    "d4rl": dict(_BASE, obs=17, act=6, hidden=(256, 256), vae_hidden=(512, 512), latent=12, size=600, bs=256, updates=3,
                 compact=True, critic2=True),
    "net": dict(_BASE, obs=5, act=3, hidden=(32, 32), vae_hidden=(24, 24), latent=6, size=120, bs=32, updates=4, per_row=True,
                critic2=True, critic2_lr=3e-4, actor_lr=3e-3, max_action=2.0, phi=3.0, lmbda=0.5, N=1, p_done=0.4, gamma=0.9,
                tau=0.05),
    "small": dict(_BASE, obs=3, act=1, hidden=(64,), vae_hidden=(32, 32), latent=2, size=200, bs=32, updates=4, max_action=2.0,
                  policy_obs=10),
}


def named(mod: torch.nn.Module, prefix: str, compact: bool) -> dict[str, np.ndarray]:
    return {f"{prefix}{i}": golden_view(p) if compact else p.detach().numpy().copy() for i, p in enumerate(mod.parameters())}


def transitions(rng, n, O, A, max_action, p_done):
    term = rng.random(n) < p_done
    trunc = (rng.random(n) < 0.03) & ~term
    term[[0, -1]], trunc[[0, -1]] = True, False
    return dict(obs=rng.standard_normal((n, O)).astype(np.float32),
                act=(max_action * np.tanh(rng.standard_normal((n, A)))).astype(np.float32), rew=rng.standard_normal(n),
                terminated=term, truncated=trunc, obs_next=rng.standard_normal((n, O)).astype(np.float32))


def build(cfg):
    O, A, H, VH, L, m = cfg["obs"], cfg["act"], cfg["hidden"], cfg["vae_hidden"], cfg["latent"], cfg["max_action"]
    if cfg["per_row"]:
        net_a = Net(state_shape=(O + A,), action_shape=(A,), hidden_sizes=H)
    else:
        net_a = MLP(input_dim=O + A, output_dim=A, hidden_sizes=H)
    pert = Perturbation(preprocess_net=net_a, max_action=m, phi=cfg["phi"])
    crit = lambda: ContinuousCritic(preprocess_net=Net(state_shape=(O,), action_shape=(A,), hidden_sizes=H, concat=True))
    c1 = crit()
    c2 = crit() if cfg["critic2"] else None
    vae = VAE(encoder=MLP(input_dim=O + A, hidden_sizes=VH), decoder=MLP(input_dim=O + L, output_dim=A, hidden_sizes=VH),
              hidden_dim=VH[-1], latent_dim=L, max_action=m)
    for k, mod in enumerate((pert, c1, c2, vae)):
        if mod is not None:
            seeded_params(mod, cfg["init_seed"] + k)
    policy = BCQPolicy(actor_perturbation=pert, critic=c1, vae=vae, action_space=Box(-m, m, (A,)),
                       forward_sampled_times=cfg["S"])
    return BCQ(policy=policy, actor_perturbation_optim=AdamOptimizerFactory(lr=cfg["actor_lr"]),
               critic_optim=AdamOptimizerFactory(lr=cfg["critic_lr"]), vae_optim=AdamOptimizerFactory(lr=cfg["vae_lr"]), critic2=c2,
               critic2_optim=AdamOptimizerFactory(lr=cfg["critic2_lr"]) if c2 is not None else None, gamma=cfg["gamma"],
               tau=cfg["tau"], lmbda=cfg["lmbda"], num_sampled_action=cfg["N"])


def gen(tag: str, cfg: dict) -> None:
    algo = build(cfg)
    out = {"cfg_" + k: np.asarray(v) for k, v in cfg.items()}
    out["state_dict_keys"] = np.asarray(sorted(algo.state_dict().keys()))
    rng = np.random.default_rng(23)
    d = transitions(rng, cfg["size"], cfg["obs"], cfg["act"], cfg["max_action"], cfg["p_done"])
    buf = ReplayBuffer.from_data(d["obs"], d["act"], d["rew"], d["terminated"], d["truncated"],
                                 np.logical_or(d["terminated"], d["truncated"]), d["obs_next"])
    for k in ("obs", "act", "rew", "terminated", "truncated", "done", "obs_next"):
        out["buf_" + k] = np.asarray(buf._meta[k]).copy()
    captured = {}
    orig_pre = algo._preprocess_batch

    def pre(batch, buffer, indices):
        captured["indices"] = np.asarray(indices).copy()
        return orig_pre(batch, buffer, indices)

    algo._preprocess_batch = pre
    c = cfg["compact"]
    nets = (("pert_", algo.policy.actor_perturbation), ("c1_", algo.policy.critic), ("c2_", algo.critic2), ("vae_", algo.policy.vae),
            ("pold_", algo.actor_perturbation_target), ("c1old_", algo.critic_target), ("c2old_", algo.critic2_target))
    for u in range(cfg["updates"]):
        np.random.seed(500 + u)
        torch.manual_seed(100 + u)
        with policy_within_training_step(algo.policy):
            stats = algo.update(buf, cfg["bs"])
        o = f"u{u}_"
        out[o + "indices"] = captured["indices"]
        out[o + "losses"] = np.array([stats.actor_loss, stats.critic1_loss, stats.critic2_loss, stats.vae_loss], dtype=np.float64)
        out[o + "torch_rng"] = torch.get_rng_state().numpy().copy()
        if c and u < cfg["updates"] - 1:
            continue        # compact: parameters after the LAST update only (every earlier step feeds into them)
        for prefix, mod in nets:
            out.update(named(mod, o + prefix, c))
    if cfg["policy_obs"]:
        obs = rng.standard_normal((cfg["policy_obs"], cfg["obs"])).astype(np.float32)
        torch.manual_seed(900)
        with torch.no_grad():
            act = algo.policy(Batch(obs=obs, info={})).act
        out["policy_obs"], out["policy_act"] = obs, np.asarray(act)
        out["policy_torch_rng"] = torch.get_rng_state().numpy().copy()
    np.savez_compressed(os.path.join(OUT, f"bcq_ref_{tag}.npz"), **out)
    print(f"bcq_ref_{tag}.npz", len(out), "arrays; losses", [out[f"u{u}_losses"].tolist() for u in range(cfg["updates"])])


if __name__ == "__main__":
    os.makedirs(OUT, exist_ok=True)
    for tag in sys.argv[1:] or list(VARIANTS):
        gen(tag, VARIANTS[tag])
