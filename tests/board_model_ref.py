"""PyTorch restatement of the board-game MuZero network: lzero/model/muzero_model.py:20-272 with downsample=False, the
reference's default and the network of its tictactoe / connect4 / gomoku configs.  The representation is conv3x3(obs -> C,
no bias) -> BN -> ReLU -> ResBlocks at board resolution (common.py:764-787); the dynamics and prediction networks are those of
the DownSample model (oracle/model_ref.py) at the board's H x W.  State-dict keys follow the reference class."""
from typing import Sequence

import torch
from torch import nn

from oracle import model_ref as R

# the shipped board configs (reference zoo/board_games/*/config), one 8x8 case with 3 blocks and 8 head channels, and the
# corners of the space lz_model_create accepts (boards up to 8x8, 1 to 16 planes, 1 to 64 actions, 1 to 4 blocks, head
# channels 1 to 16, head hidden 1 to 32, supports up to 608):
# name -> (observation_shape, A, C, blocks, head channels, head hidden, support range); head channels and hidden sizes are
# one value for the three heads or a (reward, value, policy) triple
BOARD_CONFIGS = {
    "tictactoe": ((3, 3, 3), 9, 16, 1, 16, 8, (-10., 11., 1.)),
    "gomoku": ((3, 6, 6), 36, 32, 1, 16, 32, (-10., 11., 1.)),
    "connect4": ((3, 6, 7), 7, 64, 1, 16, 32, (-300., 301., 1.)),
    "board8x8_r3": ((2, 8, 8), 64, 64, 3, 8, 32, (-10., 11., 1.)),
    # a one-row board (the +-(W + 2)-row tap shifts read only pad rows), 16 planes, one action, 4 blocks (17 layers, the weight
    # ring wraps over 153 taps), reward and policy heads of one channel and one hidden unit, 608 support bins
    "row1x8_r4": ((16, 1, 8), 1, 16, 4, (1, 16, 1), (1, 32, 1), (-304., 304., 1.)),
    # a one-column board (the +-1 tap shifts read only the pad column), one observation plane
    "col8x1": ((1, 8, 1), 8, 32, 2, 4, 8, (-10., 11., 1.)),
    # 16 head channels on an 8x8 board (FC1 over 1024 inputs), 64 actions, 4 blocks, up to 8 tiles of 16 channels
    "board8x8_hc16": ((5, 8, 8), 64, 16, 4, 16, (32, 1, 32), (-300., 301., 1.)),
}


class BoardRepresentationNetwork(nn.Module):
    """lzero/model/common.py:706-787 with downsample=False, norm_type='BN', use_sim_norm=False"""

    def __init__(self, observation_shape, num_res_blocks, num_channels):
        super().__init__()
        self.conv = nn.Conv2d(observation_shape[0], num_channels, kernel_size=3, stride=1, padding=1, bias=False)
        self.norm = nn.BatchNorm2d(num_channels)
        self.resblocks = nn.ModuleList([R.ResBlock(num_channels) for _ in range(num_res_blocks)])

    def forward(self, x):
        x = torch.relu(self.norm(self.conv(x)))
        for b in self.resblocks:
            x = b(x)
        return x


class BoardMuZeroModelRef(R.MuZeroModelRef):
    """MuZeroModelRef's initial / recurrent inference on the full-resolution board network"""

    def __init__(self, observation_shape: Sequence[int] = (3, 3, 3), action_space_size: int = 9, num_res_blocks: int = 1,
                 num_channels: int = 16, reward_head_channels: int = 16, value_head_channels: int = 16,
                 policy_head_channels: int = 16, reward_head_hidden_channels=(32,), value_head_hidden_channels=(32,),
                 policy_head_hidden_channels=(32,), reward_support_range=(-300., 301., 1.), value_support_range=(-300., 301., 1.),
                 last_linear_layer_init_zero: bool = True):
        nn.Module.__init__(self)
        self.action_space_size = action_space_size
        self.reward_support_size = len(torch.arange(*reward_support_range))
        self.value_support_size = len(torch.arange(*value_support_range))
        H, W = observation_shape[1], observation_shape[2]
        self.latent_hw = (H, W)
        P = H * W
        self.representation_network = BoardRepresentationNetwork(observation_shape, num_res_blocks, num_channels)
        self.dynamics_network = R.DynamicsNetwork(
            action_space_size, num_res_blocks, num_channels, reward_head_channels, list(reward_head_hidden_channels),
            self.reward_support_size, reward_head_channels * P, last_linear_layer_init_zero)
        self.prediction_network = R.PredictionNetwork(
            action_space_size, num_res_blocks, num_channels, value_head_channels, policy_head_channels,
            list(value_head_hidden_channels), list(policy_head_hidden_channels), self.value_support_size,
            value_head_channels * P, policy_head_channels * P, last_linear_layer_init_zero)


def config(name):
    """BOARD_CONFIGS[name], or `name` itself when it is a config tuple"""
    return BOARD_CONFIGS[name] if isinstance(name, str) else name


def model_kwargs(name):
    """constructor keywords of config `name` (a BOARD_CONFIGS key or a config tuple), as a board config passes them to
    MuZeroModel"""
    obs, A, C, nres, hc, hid, sup = config(name)
    hc = (hc,) * 3 if isinstance(hc, int) else hc
    hid = (hid,) * 3 if isinstance(hid, int) else hid
    return dict(observation_shape=obs, action_space_size=A, num_res_blocks=nres, num_channels=C, reward_head_channels=hc[0],
                value_head_channels=hc[1], policy_head_channels=hc[2], reward_head_hidden_channels=[hid[0]],
                value_head_hidden_channels=[hid[1]], policy_head_hidden_channels=[hid[2]], reward_support_range=sup,
                value_support_range=sup)


def build(name, seed):
    """the restatement of config `name` with seeded, non-degenerate (emulate_trained_) weights"""
    torch.manual_seed(seed)
    return live_single_units_(R.emulate_trained_(BoardMuZeroModelRef(**model_kwargs(name)), seed))


@torch.no_grad()
def live_single_units_(model):
    """A head of one channel or one hidden unit funnels through a single ReLU, which random weights leave dead for every input
    about half the time: the head's logits are then its FC2 bias whatever the latent, and a wrong head path goes unseen.  Such
    a unit reads only ReLU outputs, so non-negative weights into it and a BN shift of +1 keep it live and input-dependent."""
    d, p = model.dynamics_network, model.prediction_network
    for conv, norm, mlp in ((d.conv1x1_reward, d.norm_reward, d.fc_reward_head), (p.conv1x1_value, p.norm_value, p.fc_value),
                            (p.conv1x1_policy, p.norm_policy, p.fc_policy)):
        for lin, bn in ((conv, norm), (mlp[0], mlp[1])):
            if bn.num_features == 1:
                lin.weight.abs_()
                bn.bias.fill_(1.0)
    return model


def board_plan(C, H, W, B):
    """(R, NT, ctas, last) of board_plan (csrc/board_tc.cu): R = B / 132 roots per CTA rounded up, capped by the rows of the
    largest tile count (8 tiles of 64 rows for C = 16 and 32, 4 for C = 64); NT the fewest tiles that hold R roots'
    (H + 1)(W + 1) rows less the last root's W + 2 trailing pad rows"""
    rpr, pad, max_tiles = (H + 1) * (W + 1), W + 2, 4 if C == 64 else 8
    R = min(max(1, (max_tiles * 64 + pad) // rpr), max(1, -(-B // 132)))
    NT = max(1, -(-(R * rpr - pad) // 64))
    ctas = -(-B // R)
    return R, NT, ctas, B - (ctas - 1) * R
