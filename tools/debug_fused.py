import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
import numpy as np, torch
from ts_testutil import PARAM_ORDER, build_ppo, load_golden, named_params, restore_vector_buffer
from test_ppo_gpu import ppo_kwargs
from tianshou_b200.utils import policy_within_training_step
g = load_golden("ppo_ref_A.npz")
algo, actor, critic = build_ppo(17, 6, "cuda:0", params={k: g["p0_" + k] for k in PARAM_ORDER}, **ppo_kwargs(g))
buf = restore_vector_buffer(g, "u0_", int(g["cfg_E"]), int(g["cfg_cap"]), device="cuda:0")
np.random.seed(1000)
p0 = algo._flat.flat.clone()
with policy_within_training_step(algo.policy):
    stats = algo.update(buffer=buf, batch_size=128, repeat=1)
torch.cuda.synchronize()
print("fused disabled:", os.environ.get("TS_B200_NO_FUSED_STEP"))
print("loss mean", stats.loss.mean, "ref", g["u0_losses"][:4, 0].mean(), "step", int(algo._flat.step_dev.item()))
print("param delta", float((algo._flat.flat - p0).abs().max()), "ref delta", float(np.abs(g["u0_p_c_w2"] - g["p0_c_w2"]).max()))
print("grad scratch extras", algo._flat.grad[-4:].cpu().numpy())
