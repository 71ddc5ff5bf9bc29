"""Pin the eager-PyTorch restatement of GAIL's discriminator half (oracle/oracle_gail.py) to outputs of the imported reference
(tests/golden/gail_ref_*.npz), and the host-side draws GAIL makes to the reference's: the discriminator's chunk bounds, the
expert buffer's index stream and numpy's global state after an update.  CPU only."""
import numpy as np
import pytest
import torch

from oracle import oracle_gail as og
from ts_testutil import load_golden, restore_vector_buffer

VARIANTS = ["gail_ref_tc", "gail_ref_merge", "gail_ref_steps", "gail_ref_layered"]


def expert_buffer(g):
    """The golden's expert buffer as a tianshou_b200 buffer (host arrays only)."""
    from tianshou_b200.data import ReplayBuffer
    if int(g["cfg_vector_expert"]):
        return restore_vector_buffer(g, "exp_", 4, 50)
    return ReplayBuffer.from_data(*(g["exp_" + k] for k in ("obs", "act", "rew", "terminated", "truncated")),
                                  g["exp_terminated"] | g["exp_truncated"], g["exp_obs_next"])


def _state(st):
    return np.asarray(st[1], dtype=np.uint32), int(st[2]), np.array([float(st[3]), float(st[4])])


def assert_generator_state(g, prefix, st):
    key, pos, gauss = _state(st)
    assert np.array_equal(key, g[prefix + "key"]) and pos == int(g[prefix + "pos"]), prefix
    assert np.array_equal(gauss, g[prefix + "gauss"]), prefix


@pytest.mark.parametrize("n,dun,sizes", [(128, 3, [42, 42, 44]), (120, 11, [10] * 12), (256, 2, [128, 128]), (10, 3, [3, 3, 4]),
                                         (7, 7, [1] * 7), (5, 2, [2, 3])])
def test_step_bounds(n, dun, sizes):
    from tianshou_b200.data.batch import minibatch_bounds
    b = og.step_bounds(n, dun)
    assert [hi - lo for lo, hi in b] == sizes
    assert b == minibatch_bounds(n, n // dun, merge_last=True)


def test_step_bounds_refuse_an_empty_chunk():
    with pytest.raises(AssertionError):
        og.step_bounds(3, 4)


@pytest.mark.parametrize("variant", VARIANTS)
def test_gail_oracle_matches_reference_run(variant):
    g = load_golden(f"{variant}.npz")
    O, A, dun = int(g["cfg_obs"]), int(g["cfg_act"]), int(g["cfg_dun"])
    hidden = tuple(int(h) for h in g["cfg_hidden"])
    disc = og.disc_net(O, A, hidden, torch.nn.ReLU if int(g["cfg_disc_relu"]) else torch.nn.Tanh)
    with torch.no_grad():
        for i, p in enumerate(disc.parameters()):
            p.copy_(torch.as_tensor(g[f"p0_disc_{i}"]).reshape(p.shape))
    opt = torch.optim.Adam(disc.parameters(), lr=float(g["cfg_disc_lr"]))
    exp = expert_buffer(g)
    vector = bool(int(g["cfg_vector_expert"]))
    exp_obs_all = g["exp_buf_obs"] if vector else g["exp_obs"]
    exp_act_all = g["exp_buf_act"] if vector else g["exp_act"]
    for u in range(2):
        o = f"u{u}_"
        N = g[o + "adv"].shape[0]
        obs = torch.as_tensor(g[o + "buf_obs"][:N])
        act = torch.as_tensor(g[o + "buf_act"][:N])
        rew = og.rewards(disc, obs, act)
        assert rew.dtype == torch.float32
        np.testing.assert_allclose(rew.double().numpy(), g[o + "rew"], rtol=1e-6, atol=1e-7, err_msg=f"{variant} u{u} rew")
        # host draws: the discriminator's order first, then the expert indices (the expert buffer's own generators)
        np.random.seed(int(g[o + "np_seed"]))
        order = np.random.permutation(N)
        bounds = og.step_bounds(N, dun)
        idx = np.concatenate([exp.sample_indices(N // dun) for _ in bounds])
        assert np.array_equal(idx, g[o + "exp_idx"]), f"{variant} u{u}: expert indices"
        for _ in range(int(g["cfg_repeat"])):        # PPO's passes draw after the discriminator
            np.random.permutation(N)
        assert_generator_state(g, o + "rng_np_", np.random.get_state())
        assert_generator_state(g, o + "rng_exp_", exp._random_state.get_state())
        if vector:
            for e in range(4):
                assert_generator_state(g, f"{o}rng_exp{e}_", exp._child_rng(e).get_state())
        for grp in opt.param_groups:
            grp["lr"] = float(g[o + "disc_lr"])
        res = og.disc_update(disc, opt, obs, act, order, torch.as_tensor(exp_obs_all[idx]), torch.as_tensor(exp_act_all[idx]), dun)
        np.testing.assert_allclose(res["loss"], g[o + "disc_loss"], rtol=1e-6, err_msg=f"{variant} u{u} disc_loss")
        assert res["acc_pi"] == list(g[o + "acc_pi"]) and res["acc_exp"] == list(g[o + "acc_exp"])
        np.testing.assert_allclose(res["margin_pi"], g[o + "margin_pi"], rtol=1e-4)
        np.testing.assert_allclose(res["margin_exp"], g[o + "margin_exp"], rtol=1e-4)
        for i, p in enumerate(disc.parameters()):
            ref = g[f"{o}disc_{i}"]
            np.testing.assert_allclose(p.detach().numpy(), ref.reshape(p.shape), rtol=1e-4, atol=1e-6,
                                       err_msg=f"{variant} u{u} disc_{i}")


@pytest.mark.parametrize("variant", VARIANTS)
def test_golden_accuracy_margins_are_away_from_zero(variant):
    """Every logit behind an accuracy count is far from 0 compared with fp32 noise, so a device run must count the same."""
    g = load_golden(f"{variant}.npz")
    for u in range(2):
        assert g[f"u{u}_margin_pi"].min() > 1e-4 and g[f"u{u}_margin_exp"].min() > 1e-4
