"""PyTorch restatement of the board Stochastic MuZero network: lzero/model/stochastic_muzero_model.py with downsample=False, the
network of the 2048 config.  Representation and prediction are the board MuZero networks (tests/board_model_ref.py).  The two
dynamics networks take [state | one encoding plane]: the afterstate dynamics a plane of value action / action_space_size, the
dynamics a plane of value chance / chance_space_size, both computed in float32 as the reference computes them.  Their conv maps
C + 1 planes to C (no bias), then bn, the state added back, ReLU, ResBlocks, and a reward head conv1x1_reward -> bn_reward ->
ReLU -> MLP.  The afterstate prediction network is a prediction network whose BNs are bn_value / bn_policy and whose policy
has chance_space_size outputs.  State-dict keys follow the reference class (chance_encoder.* aside, which inference never
reads).  tests/golden/make_stochastic_board_golden.py pins it bit for bit to the reference class and writes
tests/golden/stoch_board_<name>.npz; the CUDA model is checked against both, in float32 and float64."""
import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import board_model_ref as BR  # noqa: E402
from oracle import model_ref as R  # noqa: E402

# name -> (observation_shape, action_space_size, chance_space_size, num_channels, blocks, head channels, head hidden, support);
# head channels and hidden sizes are one value for the three heads or a (reward, value, policy) triple
CONFIGS = {
    # zoo/game_2048/config/stochastic_muzero_2048_config.py: the model's defaults with its observation, 4 actions, 16 cells x 2
    # tiles of chance outcomes and the (0, 601) support
    "game_2048": ((16, 4, 4), 4, 32, 64, 1, 16, 32, (0., 601., 1.)),
    # the corners of lz_model_create_stochastic: C = 16 on 3x3 with one chance outcome
    "c16_3x3_ch1": ((3, 3, 3), 9, 1, 16, 1, 16, 8, (-10., 11., 1.)),
    # C = 32 on a non-square 6x7 board with more chance outcomes than actions, reward and policy heads of one channel
    "c32_6x7_ch20": ((3, 6, 7), 7, 20, 32, 1, (1, 16, 1), 32, (-300., 301., 1.)),
    # the same board with more actions than chance outcomes, two blocks, a value head of one hidden unit
    "c32_6x7_a12": ((5, 6, 7), 12, 5, 32, 2, 8, (32, 1, 32), (-10., 11., 1.)),
    # 4 ResBlocks per network: 17 layers in each recurrent program
    "c16_5x5_r4": ((4, 5, 5), 6, 3, 16, 4, 8, 16, (-300., 301., 1.)),
    # 8x8 at C = 64 with 64 chance outcomes and 64 actions
    "c64_8x8_ch64": ((2, 8, 8), 64, 64, 64, 1, 16, 32, (-10., 11., 1.)),
}


def _triple(x):
    return (x,) * 3 if isinstance(x, int) else tuple(x)


class StochasticDynamicsNetwork(nn.Module):
    """stochastic_muzero_model.py:481-577 (DynamicsNetwork, and AfterstateDynamicsNetwork, the same class); `num_channels` is the
    latent's C (the reference's num_channels - 1)"""

    def __init__(self, num_res_blocks, num_channels, reward_head_channels, reward_hidden, support_size, flatten_size):
        super().__init__()
        self.conv = nn.Conv2d(num_channels + 1, num_channels, 3, 1, 1, bias=False)
        self.bn = nn.BatchNorm2d(num_channels)
        self.resblocks = nn.ModuleList([R.ResBlock(num_channels) for _ in range(num_res_blocks)])
        self.conv1x1_reward = nn.Conv2d(num_channels, reward_head_channels, 1)
        self.bn_reward = nn.BatchNorm2d(reward_head_channels)
        self.fc_reward_head = R.MLP_V2(flatten_size, [reward_hidden], support_size)

    def forward(self, state_encoding):
        x = torch.relu(self.bn(self.conv(state_encoding)) + state_encoding[:, :-1])
        for b in self.resblocks:
            x = b(x)
        r = torch.relu(self.bn_reward(self.conv1x1_reward(x)))
        return x, self.fc_reward_head(r.reshape(r.shape[0], -1))


class AfterstatePredictionNetwork(nn.Module):
    """stochastic_muzero_model.py:580-683"""

    def __init__(self, chance_space_size, num_res_blocks, num_channels, value_head_channels, policy_head_channels,
                 value_hidden, policy_hidden, support_size, flat_value, flat_policy):
        super().__init__()
        self.resblocks = nn.ModuleList([R.ResBlock(num_channels) for _ in range(num_res_blocks)])
        self.conv1x1_value = nn.Conv2d(num_channels, value_head_channels, 1)
        self.conv1x1_policy = nn.Conv2d(num_channels, policy_head_channels, 1)
        self.bn_value = nn.BatchNorm2d(value_head_channels)
        self.bn_policy = nn.BatchNorm2d(policy_head_channels)
        self.fc_value = R.MLP_V2(flat_value, [value_hidden], support_size)
        self.fc_policy = R.MLP_V2(flat_policy, [policy_hidden], chance_space_size)

    def forward(self, x):
        for b in self.resblocks:
            x = b(x)
        v = torch.relu(self.bn_value(self.conv1x1_value(x)))
        p = torch.relu(self.bn_policy(self.conv1x1_policy(x)))
        return self.fc_policy(p.reshape(p.shape[0], -1)), self.fc_value(v.reshape(v.shape[0], -1))


class StochasticMuZeroModelRef(nn.Module):
    def __init__(self, observation_shape, action_space_size, chance_space_size, num_channels, num_res_blocks, head_channels,
                 head_hidden, support_range):
        super().__init__()
        hc, hid = _triple(head_channels), _triple(head_hidden)
        K = len(torch.arange(*support_range))
        P = observation_shape[1] * observation_shape[2]
        self.action_space_size, self.chance_space_size = action_space_size, chance_space_size
        self.representation_network = BR.BoardRepresentationNetwork(observation_shape, num_res_blocks, num_channels)
        self.dynamics_network = StochasticDynamicsNetwork(num_res_blocks, num_channels, hc[0], hid[0], K, hc[0] * P)
        self.prediction_network = R.PredictionNetwork(action_space_size, num_res_blocks, num_channels, hc[1], hc[2], [hid[1]],
                                                      [hid[2]], K, hc[1] * P, hc[2] * P)
        self.afterstate_dynamics_network = StochasticDynamicsNetwork(num_res_blocks, num_channels, hc[0], hid[0], K, hc[0] * P)
        self.afterstate_prediction_network = AfterstatePredictionNetwork(chance_space_size, num_res_blocks, num_channels, hc[1],
                                                                         hc[2], hid[1], hid[2], K, hc[1] * P, hc[2] * P)

    def initial_inference(self, obs):
        latent = self.representation_network(obs)
        policy_logits, value = self.prediction_network(latent)
        return R.MZNetworkOutput(value, [0. for _ in range(obs.size(0))], policy_logits, latent)

    def recurrent_inference(self, state, option, afterstate=False):
        """stochastic_muzero_model.py:233-273; the encoding plane's value option / n is rounded to float32 as the reference's
        is, whatever the state's dtype"""
        n = self.chance_space_size if afterstate else self.action_space_size
        B, _, H, W = state.shape
        ones = torch.ones(B, 1, H, W, device=state.device)
        plane = (option.to(state.device).reshape(B, 1, 1, 1).float() * ones / n).to(state.dtype)
        x = torch.cat((state, plane), dim=1)
        if afterstate:
            nxt, reward = self.dynamics_network(x)
            policy_logits, value = self.prediction_network(nxt)
        else:
            nxt, reward = self.afterstate_dynamics_network(x)
            policy_logits, value = self.afterstate_prediction_network(nxt)
        return R.MZNetworkOutput(value, reward, policy_logits, nxt)


def model_kwargs(name):
    """constructor keywords of config `name` as the reference's StochasticMuZeroModel takes them"""
    obs, A, NC, C, nres, hc, hid, sup = CONFIGS[name]
    hc, hid = _triple(hc), _triple(hid)
    return dict(observation_shape=obs, action_space_size=A, chance_space_size=NC, num_res_blocks=nres, num_channels=C,
                reward_head_channels=hc[0], value_head_channels=hc[1], policy_head_channels=hc[2],
                reward_head_hidden_channels=[hid[0]], value_head_hidden_channels=[hid[1]], policy_head_hidden_channels=[hid[2]],
                reward_support_range=sup, value_support_range=sup)


@torch.no_grad()
def live_single_units_(model):
    """board_model_ref.live_single_units_ for the five heads: a head of one channel or one hidden unit gets non-negative
    weights into that unit and a BN shift of +1, so it stays live and input-dependent"""
    pairs = []
    for d in (model.dynamics_network, model.afterstate_dynamics_network):
        pairs.append((d.conv1x1_reward, d.bn_reward, d.fc_reward_head))
    p, a = model.prediction_network, model.afterstate_prediction_network
    pairs += [(p.conv1x1_value, p.norm_value, p.fc_value), (p.conv1x1_policy, p.norm_policy, p.fc_policy),
              (a.conv1x1_value, a.bn_value, a.fc_value), (a.conv1x1_policy, a.bn_policy, a.fc_policy)]
    for conv, norm, mlp in pairs:
        for lin, bn in ((conv, norm), (mlp[0], mlp[1])):
            if bn.num_features == 1:
                lin.weight.abs_()
                bn.bias.fill_(1.0)
    return model


def build(name, seed, dtype=torch.float32):
    """the restatement of config `name` with seeded, non-degenerate (emulate_trained_) weights"""
    torch.manual_seed(seed)
    return live_single_units_(R.emulate_trained_(StochasticMuZeroModelRef(*CONFIGS[name]), seed)).to(dtype).eval()
