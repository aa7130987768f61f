"""PyTorch restatement of the board-game MuZero network: lzero/model/muzero_model.py:20-272 with downsample=False, the
reference's default and the network of its tictactoe / connect4 / gomoku configs.  The representation is conv3x3(obs -> C,
no bias) -> BN -> ReLU -> ResBlocks at board resolution (common.py:764-787); the dynamics and prediction networks are those of
the DownSample model (oracle/model_ref.py) at the board's H x W.  State-dict keys follow the reference class."""
from typing import Sequence

import torch
from torch import nn

from oracle import model_ref as R

# the shipped board configs (reference zoo/board_games/*/config) and one 8x8 case with 3 blocks and 8 head channels:
# name -> (observation_shape, A, C, blocks, head channels, head hidden, support range)
BOARD_CONFIGS = {
    "tictactoe": ((3, 3, 3), 9, 16, 1, 16, 8, (-10., 11., 1.)),
    "gomoku": ((3, 6, 6), 36, 32, 1, 16, 32, (-10., 11., 1.)),
    "connect4": ((3, 6, 7), 7, 64, 1, 16, 32, (-300., 301., 1.)),
    "board8x8_r3": ((2, 8, 8), 64, 64, 3, 8, 32, (-10., 11., 1.)),
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


def model_kwargs(name):
    """constructor keywords of BOARD_CONFIGS[name], as a board config passes them to MuZeroModel"""
    obs, A, C, nres, hc, hid, sup = BOARD_CONFIGS[name]
    return dict(observation_shape=obs, action_space_size=A, num_res_blocks=nres, num_channels=C, reward_head_channels=hc,
                value_head_channels=hc, policy_head_channels=hc, reward_head_hidden_channels=[hid],
                value_head_hidden_channels=[hid], policy_head_hidden_channels=[hid], reward_support_range=sup,
                value_support_range=sup)


def build(name, seed):
    """the restatement of config `name` with seeded, non-degenerate (emulate_trained_) weights"""
    torch.manual_seed(seed)
    return R.emulate_trained_(BoardMuZeroModelRef(**model_kwargs(name)), seed)
