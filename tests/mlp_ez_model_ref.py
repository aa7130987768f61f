"""PyTorch restatement of the reference's EfficientZeroModelMLP (lzero/model/efficientzero_model_mlp.py:16-300) in eval mode:
one_hot actions, categorical supports, norm_type='BN', state_norm=False, no SSL heads.  The representation and prediction
networks are MuZeroModelMLP's (oracle/model_ref.py); the dynamics network is DynamicsNetworkMLP (:345-468): fc_dynamics, or
fc_dynamics_1 + latent -> fc_dynamics_2 with res_connection_in_dynamics, then nn.LSTM(L -> H) on the dynamics output and
fc_reward_head straight on h' (no norm_value_prefix).  tests/golden/make_mlp_ez_golden.py pins it bit for bit to the reference
class; the CUDA model is checked against both."""
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.model_ref import (DingMLP, EZNetworkOutput, PredictionNetworkMLP, RepresentationNetworkMLP,  # noqa: E402
                              emulate_trained_mlp_)

# name -> (observation_shape, action_space_size, latent_state_dim, lstm_hidden_size, res_connection_in_dynamics)
CONFIGS = {
    "cartpole": (4, 2, 128, 128, False),            # zoo/classic_control/cartpole/config/cartpole_efficientzero_config.py
    "lunarlander": (8, 4, 256, 256, True),          # zoo/box2d/lunarlander/config/lunarlander_disc_efficientzero_config.py
    "minigrid": (2835, 7, 256, 256, False),         # zoo/minigrid/config/minigrid_efficientzero_config.py
    "bipedalwalker": (24, 256, 256, 256, True),     # zoo/box2d/bipedalwalker/config/bipedalwalker_cont_disc_efficientzero_config.py
    "defaults": (2, 6, 256, 512, False),            # the class defaults (efficientzero_model_mlp.py:16-40)
    "l96_h48": (5, 3, 96, 48, False),               # a shape of the fp32 LSTM kernel (k_ez_lstm: L, H not multiples of 64)
    # the narrowest latent (k_mez_tc<1>) on a one-feature observation
    "l32_o1": (1, 5, 32, 32, False),
    # k_mez_tc<2> on the widest observation: 128 streamed 32-feature chunks
    "l64_o4096": (4096, 3, 64, 64, True),
    # k_mez_tc<6>
    "l192": (40, 9, 192, 96, False),
}


def model_kwargs(name):
    obs, A, L, H, res = CONFIGS[name]
    return dict(observation_shape=obs, action_space_size=A, latent_state_dim=L, lstm_hidden_size=H,
                res_connection_in_dynamics=res)


class DynamicsNetworkMLPEZ(nn.Module):
    """efficientzero_model_mlp.py:345-468 with norm_type='BN' and ReLU"""

    def __init__(self, A, L, H, reward_hidden, support_size, res):
        super().__init__()
        self.action_encoding_dim = A
        self.res_connection_in_dynamics = res
        if res:
            self.fc_dynamics_1 = DingMLP(L + A, L, L, 2)
            self.fc_dynamics_2 = DingMLP(L, L, L, 2)
        else:
            self.fc_dynamics = DingMLP(L + A, L, L, 2)
        self.lstm = nn.LSTM(input_size=L, hidden_size=H)
        self.fc_reward_head = DingMLP(H, reward_hidden, support_size, 2, output_activation=False, output_norm=False)

    def forward(self, sa, hidden):
        if self.res_connection_in_dynamics:
            nxt = self.fc_dynamics_1(sa) + sa[:, :-self.action_encoding_dim]
            enc = self.fc_dynamics_2(nxt)
        else:
            nxt = self.fc_dynamics(sa)
            enc = nxt
        y, hidden = self.lstm(enc.unsqueeze(0), hidden)
        return nxt, hidden, self.fc_reward_head(y.squeeze(0)), enc


class EfficientZeroModelMLPRef(nn.Module):
    def __init__(self, observation_shape=2, action_space_size=6, latent_state_dim=256, lstm_hidden_size=512,
                 reward_head_hidden_channels=(32,), value_head_hidden_channels=(32,), policy_head_hidden_channels=(32,),
                 reward_support_range=(-300., 301., 1.), value_support_range=(-300., 301., 1.), res_connection_in_dynamics=False):
        super().__init__()
        self.action_space_size = action_space_size
        self.lstm_hidden_size = lstm_hidden_size
        K = len(torch.arange(*value_support_range))
        self.representation_network = RepresentationNetworkMLP(observation_shape, latent_state_dim)
        self.dynamics_network = DynamicsNetworkMLPEZ(action_space_size, latent_state_dim, lstm_hidden_size,
                                                     reward_head_hidden_channels[0], len(torch.arange(*reward_support_range)),
                                                     res_connection_in_dynamics)
        self.prediction_network = PredictionNetworkMLP(action_space_size, latent_state_dim, value_head_hidden_channels,
                                                       policy_head_hidden_channels, K)

    def initial_inference(self, obs):
        B = obs.size(0)
        latent = self.representation_network(obs)
        policy_logits, value = self.prediction_network(latent)
        hidden = (torch.zeros(1, B, self.lstm_hidden_size), torch.zeros(1, B, self.lstm_hidden_size))
        return EZNetworkOutput(value, [0. for _ in range(B)], policy_logits, latent, hidden)

    def one_hot(self, action):
        if action.dim() == 1:
            action = action.unsqueeze(-1)
        oh = torch.zeros(action.shape[0], self.action_space_size, device=action.device)
        oh.scatter_(1, action.long(), 1)
        return oh

    def recurrent_inference(self, latent_state, reward_hidden_state, action):
        nxt, hidden, value_prefix, _ = self.dynamics_network(torch.cat((latent_state, self.one_hot(action).float()), dim=1),
                                                             reward_hidden_state)
        policy_logits, value = self.prediction_network(nxt)
        return EZNetworkOutput(value, value_prefix, policy_logits, nxt, hidden)

    def lstm_input(self, latent_state, action):
        """the dynamics network's output that enters the LSTM"""
        return self.dynamics_network(torch.cat((latent_state, self.one_hot(action).float()), dim=1), None)[3]


def build(name, seed, dtype=torch.float32):
    torch.manual_seed(seed)
    m = emulate_trained_mlp_(EfficientZeroModelMLPRef(**model_kwargs(name)), seed)
    g = torch.Generator().manual_seed(seed + 1000)
    with torch.no_grad():      # LSTM weights of a trained scale (torch's default U(-1/sqrt(H), 1/sqrt(H)) already is one)
        for p in m.dynamics_network.lstm.parameters():
            p.add_(0.02 * torch.randn(p.shape, generator=g))
    return m.to(dtype).eval()
