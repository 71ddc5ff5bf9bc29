"""Helpers shared by the CPU tests that pin the discrete Q-learning restatements under oracle/ to the reference's goldens."""
import numpy as np
import torch

from oracle import oracle_discrete_bcq as odb
from oracle import oracle_discrete_sac as ods


def oracle_setup(g, outs, device="cpu"):
    """Oracle networks with the golden's initial weights, and its buffer view and observation reader."""
    nets = odb.nets_from_cfg(g, outs)
    if bool(g["cfg_compact"]):
        ods.seeded_params(nets, int(g["cfg_init_seed"]))
    else:
        with torch.no_grad():
            for i, p in enumerate(nets.parameters()):
                p.copy_(torch.as_tensor(g[f"p0_{i}"]).reshape(p.shape))
    nets.to(device)
    E, cap = int(g["cfg_E"]), int(g["cfg_cap"])
    buf = dict(obs=g["buf_obs"], act=g["buf_act"], rew=g["buf_rew"], done=g["buf_done"], terminated=g["buf_terminated"],
               offset=np.arange(E + 1) * cap, last_index=g["meta_last_index"], lengths=g["meta_lengths"])
    if "buf_obs_next" in g:
        buf["obs_next"] = g["buf_obs_next"]
        obs_of = ods.flat_obs(buf["obs"], device)
    else:
        obs_of = ods.frame_obs(buf, 4, 255.0, device)
    return nets, buf, obs_of


def check_final(g, params, opt, lagged):
    """Final parameters, Adam moments and lagged parameters against the golden: Adam normalises a step to ~lr per element, so
    the absolute term is stated in units of one step (DESIGN.md section 4)."""
    view = ods.golden_view if bool(g["cfg_compact"]) else (lambda t: t.detach().cpu().numpy())
    lr = float(g["cfg_lr"])
    for i, p in enumerate(params):
        np.testing.assert_allclose(view(p), g[f"pf_{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"parameter {i}")
        st = opt.state[p]
        m, v = g[f"m_{i}"], g[f"v_{i}"]
        np.testing.assert_allclose(view(st["exp_avg"]), m, rtol=1e-3, atol=1e-3 * float(np.abs(m).max()) + 1e-12, err_msg=f"exp_avg {i}")
        np.testing.assert_allclose(view(st["exp_avg_sq"]), v, rtol=2e-3, atol=2e-3 * float(np.abs(v).max()) + 1e-20, err_msg=f"exp_avg_sq {i}")
        assert int(st["step"]) == int(g["adam_step"])
    for i, p in enumerate(lagged):
        np.testing.assert_allclose(view(p), g[f"old_{i}"], rtol=1e-3, atol=0.1 * lr, err_msg=f"lagged parameter {i}")
