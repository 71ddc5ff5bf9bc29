"""Which path every actor-critic takes, and its flat parameter layout: ``parse_actor_critic`` + ``fused_descriptor``
(algorithm/layered.py) over a grid of models built from the package's own module classes.  CPU only -- the parse
allocates nothing.

Each row asserts the path (fused kernels, layer-wise path, or refused), then for fused rows every ``ActorCriticDesc`` field
and the flat-buffer parameter order, for layer-wise rows the trunk sharing and the parameter order of each ``FlatGroup``,
and for refused rows a part of the message.  The sharing rows pin the rule that trunk sharing follows parameter identity:
two ``Net`` wrappers around one MLP share the trunk on either path, and a trunk that shares only some of its layers is
refused (its two backward passes would overwrite each other's gradient in the shared slots)."""
import re

import pytest
import torch
from torch import nn

DESC_FIELDS = ("obs_dim", "act_dim", "hidden", "flags", "a_w1", "a_b1", "a_w2", "a_b2", "a_w3", "a_b3", "a_logstd",
               "c_w1", "c_b1", "c_w2", "c_b2", "c_w3", "c_b3", "n_params")

OBS = (1, 17, 32, 33, 64, 65, 376)
ACTS = (1, 6, 16, 17)
HIDDEN = ((64, 64), (128, 128), (64, 64, 64))
ACTIVATION = {"tanh": nn.Tanh, "relu": nn.ReLU}


def _net(obs, hidden, act="tanh", **kw):
    from tianshou_b200.utils.net.common import Net
    return Net(state_shape=(obs,), hidden_sizes=hidden, activation=ACTIVATION[act], **kw)


def gaussian(obs, act_dim, hidden, act="tanh", *, critic_act=None, unbounded=True, conditioned_sigma=False,
             obs_only=False, share=None, **net_kw):
    """``share``: None (separate trunks), "wrap" (two Net wrappers around one MLP), "partial" (the critic trunk reuses
    the actor trunk's first Linear)."""
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.continuous import ContinuousActorProbabilistic, ContinuousCritic
    torch.manual_seed(0)
    a_net = _net(obs, hidden, act, **net_kw)
    c_net = _net(obs, hidden, critic_act or act, **net_kw)
    if share == "wrap":
        c_net = Net(state_shape=(obs,), hidden_sizes=())
        c_net.model = a_net.model
        c_net.output_dim = a_net.output_dim
    elif share == "partial":
        c_net.model.model[0] = a_net.model.model[0]
    actor = ContinuousActorProbabilistic(preprocess_net=a_net, action_shape=(act_dim,), unbounded=unbounded,
                                         conditioned_sigma=conditioned_sigma)
    critic = ContinuousCritic(preprocess_net=c_net, apply_preprocess_net_to_obs_only=obs_only)
    return actor, critic


def categorical(obs, act_dim, hidden, shared, act="relu", *, softmax_output=True, share=None, **net_kw):
    from tianshou_b200.utils.net.common import Net
    from tianshou_b200.utils.net.discrete import DiscreteActor, DiscreteCritic
    torch.manual_seed(0)
    a_net = _net(obs, hidden, act, **net_kw)
    c_net = a_net if shared else _net(obs, hidden, act, **net_kw)
    if share == "wrap":
        c_net = Net(state_shape=(obs,), hidden_sizes=())
        c_net.model = a_net.model
        c_net.output_dim = a_net.output_dim
    actor = DiscreteActor(preprocess_net=a_net, action_shape=(act_dim,), softmax_output=softmax_output)
    critic = DiscreteCritic(preprocess_net=c_net)
    return actor, critic


def grid():
    """row id -> (builder, split)."""
    rows = {}
    for act in ACTIVATION:
        for hidden in HIDDEN:
            for obs in OBS:
                for a in ACTS:
                    hid = "x".join(map(str, hidden))
                    rows[f"gauss-{act}-{hid}-obs{obs}-act{a}"] = (lambda o=obs, a=a, h=hidden, f=act: gaussian(o, a, h, f), False)
    for shared in (True, False):
        for a in (2, 6, 16, 17, 64, 65):
            rows[f"cat-{'shared' if shared else 'separate'}-act{a}"] = (lambda a=a, s=shared: categorical(4, a, (64, 64), s), False)
    rows["gauss-tanh-actor-relu-critic"] = (lambda: gaussian(17, 6, (64, 64), "tanh", critic_act="relu"), False)
    rows["gauss-conditioned-sigma"] = (lambda: gaussian(17, 6, (64, 64), conditioned_sigma=True), False)
    rows["gauss-bounded"] = (lambda: gaussian(17, 6, (64, 64), unbounded=False), False)
    rows["gauss-softmax-trunk"] = (lambda: gaussian(17, 6, (64, 64), softmax=True), False)
    rows["gauss-preprocess-obs-only"] = (lambda: gaussian(17, 6, (64, 64), obs_only=True), False)
    rows["gauss-layernorm-trunk"] = (lambda: gaussian(17, 6, (64, 64), norm_layer=nn.LayerNorm), False)
    rows["gauss-net-action-shape-trunk"] = (lambda: gaussian(17, 6, (64, 64), action_shape=(32,)), False)
    rows["cat-net-action-shape-trunk"] = (lambda: categorical(4, 2, (64, 64), True, action_shape=(16,)), False)
    rows["cat-logits-output"] = (lambda: categorical(4, 2, (64, 64), False, softmax_output=False), False)
    rows["split-gauss-separate"] = (lambda: gaussian(17, 6, (64, 64)), True)
    rows["split-gauss-wide"] = (lambda: gaussian(376, 17, (128, 128)), True)
    rows["split-cat-separate"] = (lambda: categorical(4, 2, (64, 64), False), True)
    rows["split-cat-shared"] = (lambda: categorical(4, 2, (64, 64), True), True)
    rows["split-gauss-conditioned-sigma"] = (lambda: gaussian(17, 6, (64, 64), conditioned_sigma=True), True)
    rows["share-cat-two-wrappers-64x64"] = (lambda: categorical(4, 2, (64, 64), False, share="wrap"), False)
    rows["share-gauss-two-wrappers-128x128"] = (lambda: gaussian(17, 6, (128, 128), share="wrap"), False)
    rows["share-gauss-two-wrappers-split"] = (lambda: gaussian(17, 6, (128, 128), share="wrap"), True)
    rows["share-gauss-partial-64x64"] = (lambda: gaussian(17, 6, (64, 64), share="partial"), False)
    rows["share-gauss-partial-128x128"] = (lambda: gaussian(17, 6, (128, 128), share="partial"), False)
    return rows


def param_names(actor, critic):
    """id(parameter) -> short name in ``ActorCritic(actor, critic)`` order (a shared parameter keeps its first name)."""
    from tianshou_b200.utils.net.common import ActorCritic
    names = {}
    for n, p in ActorCritic(actor, critic).named_parameters(remove_duplicate=False):
        n = n.replace("preprocess.model.model.", "trunk.").replace(".model.", ".")
        names.setdefault(id(p), n)
    return names


CAT_SHARED_NET_ACTION_SHAPE = (
    'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.trunk.4.weight', 'actor.trunk.4.bias', 'actor.last.0.weight', 'actor.last.0.bias',
    'critic.last.0.weight', 'critic.last.0.bias',
)
CAT_SEPARATE = (
    'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.last.0.weight', 'actor.last.0.bias', 'critic.trunk.0.weight', 'critic.trunk.0.bias',
    'critic.trunk.2.weight', 'critic.trunk.2.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
CAT_SHARED = (
    'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.last.0.weight', 'actor.last.0.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
GAUSS_THREE_LAYERS = (
    'actor.sigma_param', 'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.trunk.4.weight', 'actor.trunk.4.bias', 'actor.mu.0.weight', 'actor.mu.0.bias', 'critic.trunk.0.weight',
    'critic.trunk.0.bias', 'critic.trunk.2.weight', 'critic.trunk.2.bias', 'critic.trunk.4.weight',
    'critic.trunk.4.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
GAUSS_MODULE_ORDER = (
    'actor.sigma_param', 'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.mu.0.weight', 'actor.mu.0.bias', 'critic.trunk.0.weight', 'critic.trunk.0.bias', 'critic.trunk.2.weight',
    'critic.trunk.2.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
GAUSS_DESC_ORDER = (
    'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias', 'actor.mu.0.weight',
    'actor.mu.0.bias', 'actor.sigma_param', 'critic.trunk.0.weight', 'critic.trunk.0.bias', 'critic.trunk.2.weight',
    'critic.trunk.2.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
GAUSS_SHARED = (
    'actor.sigma_param', 'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.mu.0.weight', 'actor.mu.0.bias', 'critic.last.0.weight', 'critic.last.0.bias',
)
CAT_ACTOR = (
    'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.last.0.weight', 'actor.last.0.bias',
)
CRITIC = (
    'critic.trunk.0.weight', 'critic.trunk.0.bias', 'critic.trunk.2.weight', 'critic.trunk.2.bias',
    'critic.last.0.weight', 'critic.last.0.bias',
)
GAUSS_ACTOR = (
    'actor.sigma_param', 'actor.trunk.0.weight', 'actor.trunk.0.bias', 'actor.trunk.2.weight', 'actor.trunk.2.bias',
    'actor.mu.0.weight', 'actor.mu.0.bias',
)

EXPECTED = {
    'cat-logits-output': ('refused', 'actor: DiscreteActor needs softmax_output=True (Categorical over probabilities)'),
    'cat-net-action-shape-trunk': ('layered', True, (CAT_SHARED_NET_ACTION_SHAPE,)),
    'cat-separate-act16': ('fused', (4, 16, 64, 3, 0, 256, 320, 4416, 4480, 5504, -1, 5520, 5776, 5840, 9936, 10000, 10064, 10065), CAT_SEPARATE),
    'cat-separate-act17': ('layered', False, (CAT_SEPARATE,)),
    'cat-separate-act2': ('fused', (4, 2, 64, 3, 0, 256, 320, 4416, 4480, 4608, -1, 4610, 4866, 4930, 9026, 9090, 9154, 9155), CAT_SEPARATE),
    'cat-separate-act6': ('fused', (4, 6, 64, 3, 0, 256, 320, 4416, 4480, 4864, -1, 4870, 5126, 5190, 9286, 9350, 9414, 9415), CAT_SEPARATE),
    'cat-separate-act64': ('layered', False, (CAT_SEPARATE,)),
    'cat-separate-act65': ('refused', 'action width > 64 unsupported'),
    'cat-shared-act16': ('fused', (4, 16, 64, 3, 0, 256, 320, 4416, 4480, 5504, -1, 0, 256, 320, 4416, 5520, 5584, 5585), CAT_SHARED),
    'cat-shared-act17': ('layered', True, (CAT_SHARED,)),
    'cat-shared-act2': ('fused', (4, 2, 64, 3, 0, 256, 320, 4416, 4480, 4608, -1, 0, 256, 320, 4416, 4610, 4674, 4675), CAT_SHARED),
    'cat-shared-act6': ('fused', (4, 6, 64, 3, 0, 256, 320, 4416, 4480, 4864, -1, 0, 256, 320, 4416, 4870, 4934, 4935), CAT_SHARED),
    'cat-shared-act64': ('layered', True, (CAT_SHARED,)),
    'cat-shared-act65': ('refused', 'action width > 64 unsupported'),
    'gauss-bounded': ('refused', 'actor: only unbounded=True (mu without tanh) is supported'),
    'gauss-conditioned-sigma': ('refused', 'actor: conditioned sigma unsupported (need state-independent sigma_param)'),
    'gauss-layernorm-trunk': ('refused', 'outside the fused layered-network family'),
    'gauss-net-action-shape-trunk': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-preprocess-obs-only': ('refused', 'critic: apply_preprocess_net_to_obs_only unsupported'),
    'gauss-relu-128x128-obs1-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs1-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs1-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs1-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs17-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs17-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs17-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs17-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs32-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs32-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs32-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs32-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs33-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs33-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs33-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs33-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs376-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs376-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs376-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs376-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs64-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs64-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs64-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs64-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs65-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs65-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs65-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-128x128-obs65-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs1-act1': ('fused', (1, 1, 64, 1, 0, 64, 128, 4224, 4288, 4352, 4353, 4354, 4418, 4482, 8578, 8642, 8706, 8707), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs1-act16': ('fused', (1, 16, 64, 1, 0, 64, 128, 4224, 4288, 5312, 5328, 5344, 5408, 5472, 9568, 9632, 9696, 9697), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs1-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs1-act6': ('fused', (1, 6, 64, 1, 0, 64, 128, 4224, 4288, 4672, 4678, 4684, 4748, 4812, 8908, 8972, 9036, 9037), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs17-act1': ('fused', (17, 1, 64, 1, 0, 1088, 1152, 5248, 5312, 5376, 5377, 5378, 6466, 6530, 10626, 10690, 10754, 10755), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs17-act16': ('fused', (17, 16, 64, 1, 0, 1088, 1152, 5248, 5312, 6336, 6352, 6368, 7456, 7520, 11616, 11680, 11744, 11745), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs17-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs17-act6': ('fused', (17, 6, 64, 1, 0, 1088, 1152, 5248, 5312, 5696, 5702, 5708, 6796, 6860, 10956, 11020, 11084, 11085), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs32-act1': ('fused', (32, 1, 64, 1, 0, 2048, 2112, 6208, 6272, 6336, 6337, 6338, 8386, 8450, 12546, 12610, 12674, 12675), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs32-act16': ('fused', (32, 16, 64, 1, 0, 2048, 2112, 6208, 6272, 7296, 7312, 7328, 9376, 9440, 13536, 13600, 13664, 13665), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs32-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs32-act6': ('fused', (32, 6, 64, 1, 0, 2048, 2112, 6208, 6272, 6656, 6662, 6668, 8716, 8780, 12876, 12940, 13004, 13005), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs33-act1': ('fused', (33, 1, 64, 1, 0, 2112, 2176, 6272, 6336, 6400, 6401, 6402, 8514, 8578, 12674, 12738, 12802, 12803), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs33-act16': ('fused', (33, 16, 64, 1, 0, 2112, 2176, 6272, 6336, 7360, 7376, 7392, 9504, 9568, 13664, 13728, 13792, 13793), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs33-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs33-act6': ('fused', (33, 6, 64, 1, 0, 2112, 2176, 6272, 6336, 6720, 6726, 6732, 8844, 8908, 13004, 13068, 13132, 13133), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs376-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs376-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs376-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs376-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs64-act1': ('fused', (64, 1, 64, 1, 0, 4096, 4160, 8256, 8320, 8384, 8385, 8386, 12482, 12546, 16642, 16706, 16770, 16771), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs64-act16': ('fused', (64, 16, 64, 1, 0, 4096, 4160, 8256, 8320, 9344, 9360, 9376, 13472, 13536, 17632, 17696, 17760, 17761), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs64-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs64-act6': ('fused', (64, 6, 64, 1, 0, 4096, 4160, 8256, 8320, 8704, 8710, 8716, 12812, 12876, 16972, 17036, 17100, 17101), GAUSS_DESC_ORDER),
    'gauss-relu-64x64-obs65-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs65-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs65-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64-obs65-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-relu-64x64x64-obs1-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs1-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs1-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs1-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs17-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs17-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs17-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs17-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs32-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs32-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs32-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs32-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs33-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs33-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs33-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs33-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs376-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs376-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs376-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs376-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs64-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs64-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs64-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs64-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs65-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs65-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs65-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-relu-64x64x64-obs65-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-softmax-trunk': ('refused', 'actor: softmax trunk output unsupported'),
    'gauss-tanh-128x128-obs1-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs1-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs1-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs1-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs17-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs17-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs17-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs17-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs32-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs32-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs32-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs32-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs33-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs33-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs33-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs33-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs376-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs376-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs376-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs376-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs64-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs64-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs64-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs64-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs65-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs65-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs65-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-128x128-obs65-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs1-act1': ('fused', (1, 1, 64, 0, 0, 64, 128, 4224, 4288, 4352, 4353, 4354, 4418, 4482, 8578, 8642, 8706, 8707), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs1-act16': ('fused', (1, 16, 64, 0, 0, 64, 128, 4224, 4288, 5312, 5328, 5344, 5408, 5472, 9568, 9632, 9696, 9697), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs1-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs1-act6': ('fused', (1, 6, 64, 0, 0, 64, 128, 4224, 4288, 4672, 4678, 4684, 4748, 4812, 8908, 8972, 9036, 9037), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs17-act1': ('fused', (17, 1, 64, 0, 0, 1088, 1152, 5248, 5312, 5376, 5377, 5378, 6466, 6530, 10626, 10690, 10754, 10755), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs17-act16': ('fused', (17, 16, 64, 0, 0, 1088, 1152, 5248, 5312, 6336, 6352, 6368, 7456, 7520, 11616, 11680, 11744, 11745), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs17-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs17-act6': ('fused', (17, 6, 64, 0, 0, 1088, 1152, 5248, 5312, 5696, 5702, 5708, 6796, 6860, 10956, 11020, 11084, 11085), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs32-act1': ('fused', (32, 1, 64, 0, 0, 2048, 2112, 6208, 6272, 6336, 6337, 6338, 8386, 8450, 12546, 12610, 12674, 12675), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs32-act16': ('fused', (32, 16, 64, 0, 0, 2048, 2112, 6208, 6272, 7296, 7312, 7328, 9376, 9440, 13536, 13600, 13664, 13665), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs32-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs32-act6': ('fused', (32, 6, 64, 0, 0, 2048, 2112, 6208, 6272, 6656, 6662, 6668, 8716, 8780, 12876, 12940, 13004, 13005), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs33-act1': ('fused', (33, 1, 64, 0, 0, 2112, 2176, 6272, 6336, 6400, 6401, 6402, 8514, 8578, 12674, 12738, 12802, 12803), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs33-act16': ('fused', (33, 16, 64, 0, 0, 2112, 2176, 6272, 6336, 7360, 7376, 7392, 9504, 9568, 13664, 13728, 13792, 13793), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs33-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs33-act6': ('fused', (33, 6, 64, 0, 0, 2112, 2176, 6272, 6336, 6720, 6726, 6732, 8844, 8908, 13004, 13068, 13132, 13133), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs376-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs376-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs376-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs376-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs64-act1': ('fused', (64, 1, 64, 0, 0, 4096, 4160, 8256, 8320, 8384, 8385, 8386, 12482, 12546, 16642, 16706, 16770, 16771), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs64-act16': ('fused', (64, 16, 64, 0, 0, 4096, 4160, 8256, 8320, 9344, 9360, 9376, 13472, 13536, 17632, 17696, 17760, 17761), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs64-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs64-act6': ('fused', (64, 6, 64, 0, 0, 4096, 4160, 8256, 8320, 8704, 8710, 8716, 12812, 12876, 16972, 17036, 17100, 17101), GAUSS_DESC_ORDER),
    'gauss-tanh-64x64-obs65-act1': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs65-act16': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs65-act17': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64-obs65-act6': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'gauss-tanh-64x64x64-obs1-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs1-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs1-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs1-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs17-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs17-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs17-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs17-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs32-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs32-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs32-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs32-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs33-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs33-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs33-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs33-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs376-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs376-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs376-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs376-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs64-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs64-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs64-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs64-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs65-act1': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs65-act16': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs65-act17': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-64x64x64-obs65-act6': ('layered', False, (GAUSS_THREE_LAYERS,)),
    'gauss-tanh-actor-relu-critic': ('layered', False, (GAUSS_MODULE_ORDER,)),
    'share-cat-two-wrappers-64x64': ('fused', (4, 2, 64, 3, 0, 256, 320, 4416, 4480, 4608, -1, 0, 256, 320, 4416, 4610, 4674, 4675), CAT_SHARED),
    'share-gauss-partial-128x128': ('refused', 'partially shared trunks are unsupported'),
    'share-gauss-partial-64x64': ('refused', 'partially shared trunks are unsupported'),
    'share-gauss-two-wrappers-128x128': ('layered', True, (GAUSS_SHARED,)),
    'share-gauss-two-wrappers-split': ('refused', 'needs separate actor and critic trunks'),
    'split-cat-separate': ('layered', False, (CAT_ACTOR, CRITIC,)),
    'split-cat-shared': ('refused', 'a critic-only optimiser (NPG / TRPO) needs separate actor and critic trunks; shared trunks are unsupported'),
    'split-gauss-conditioned-sigma': ('refused', 'actor: conditioned sigma unsupported (need state-independent sigma_param)'),
    'split-gauss-separate': ('layered', False, (GAUSS_ACTOR, CRITIC,)),
    'split-gauss-wide': ('layered', False, (GAUSS_ACTOR, CRITIC,)),
}


ROWS = grid()


@pytest.mark.parametrize("row", sorted(EXPECTED))
def test_actor_critic_path_and_layout(row):
    from tianshou_b200.algorithm.flat_params import UnsupportedModelError
    from tianshou_b200.algorithm.layered import fused_descriptor, parse_actor_critic
    build, split = ROWS[row]
    actor, critic = build()
    expected = EXPECTED[row]
    if expected[0] == "refused":
        with pytest.raises(UnsupportedModelError, match=re.escape(expected[1])):
            parse_actor_critic(actor, critic, split=split)
        return
    names = param_names(actor, critic)
    spec = parse_actor_critic(actor, critic, split=split)
    fused = None if split else fused_descriptor(spec)
    assert ("fused" if fused is not None else "layered") == expected[0]
    if fused is not None:
        desc, params = fused
        assert tuple(getattr(desc, f) for f in DESC_FIELDS) == expected[1]
        assert tuple(names[id(p)] for p in params) == expected[2]
    else:
        assert spec.shared == expected[1]
        assert tuple(tuple(names[id(p)] for p in g) for g in spec.group_params) == expected[2]


def test_grid_is_complete():
    assert set(ROWS) == set(EXPECTED)
