"""StochasticMuZeroModelMLP (lzero/model/stochastic_muzero_model_mlp.py) restated from the MuZeroModelMLP restatement
(oracle.model_ref.MuZeroModelMLPRef): afterstate_dynamics_network is a MuZeroModelMLP dynamics network over [latent | one-hot
action], dynamics_network one over [afterstate | one-hot chance outcome], afterstate_prediction_network a prediction network with
chance_space_size outputs.  tests/golden/make_stochastic_mlp_golden.py pins it bit for bit to the reference class and writes
tests/golden/stoch_mlp_<name>.npz; the CUDA model is checked against both, in float32 and float64."""
import os
import sys

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.model_ref import MuZeroModelMLPRef, MZNetworkOutput, emulate_trained_mlp_  # noqa: E402

# name -> (observation_shape, action_space_size, chance_space_size, latent_state_dim, res_connection_in_dynamics, head hidden,
# support range)
CONFIGS = {
    # zoo/classic_control/cartpole/config/cartpole_stochastic_muzero_config.py
    "cartpole": (4, 2, 3, 128, False, 32, (-300., 301., 1.)),
    # zoo/box2d/lunarlander/config/lunarlander_disc_stochastic_muzero_config.py
    "lunarlander_disc": (8, 4, 2, 256, True, 32, (-300., 301., 1.)),
    # zoo/classic_control/pendulum/config/pendulum_cont_disc_stochastic_muzero_config.py (chance_space_size: the model default)
    "pendulum_cont_disc": (3, 11, 2, 128, False, 32, (-300., 301., 1.)),
    # the envelope's corners: latent 32, one chance outcome, head hidden layers of one unit, the residual dynamics
    "l32_c1_h1": (6, 5, 1, 32, True, 1, (-10., 11., 1.)),
    # latent 256 with the largest chance space the kernel takes (608 outcomes: 8 policy pieces of the afterstate program)
    "l256_c608": (10, 3, 608, 256, False, 32, (-300., 301., 1.)),
    # a chance space wider than the action space at a middle latent, hidden layers of 16
    "l64_c9_res": (5, 4, 9, 64, True, 16, (-300., 301., 1.)),
}


class StochasticMuZeroModelMLPRef(nn.Module):
    def __init__(self, observation_shape, action_space_size, chance_space_size, latent_state_dim, res_connection_in_dynamics,
                 hidden, support_range):
        super().__init__()
        kw = dict(latent_state_dim=latent_state_dim, reward_head_hidden_channels=(hidden,), value_head_hidden_channels=(hidden,),
                  policy_head_hidden_channels=(hidden,), reward_support_range=support_range,
                  value_support_range=support_range, res_connection_in_dynamics=res_connection_in_dynamics)
        a = MuZeroModelMLPRef(observation_shape, action_space_size, **kw)
        c = MuZeroModelMLPRef(observation_shape, chance_space_size, **kw)
        self.action_space_size, self.chance_space_size = action_space_size, chance_space_size
        self.representation_network = a.representation_network
        self.prediction_network = a.prediction_network
        self.afterstate_dynamics_network = a.dynamics_network
        self.dynamics_network = c.dynamics_network
        self.afterstate_prediction_network = c.prediction_network

    def initial_inference(self, obs):
        latent = self.representation_network(obs)
        policy_logits, value = self.prediction_network(latent)
        return MZNetworkOutput(value, [0. for _ in range(obs.size(0))], policy_logits, latent)

    def recurrent_inference(self, state, option, afterstate=False):
        """stochastic_muzero_model.py:233-273"""
        n = self.chance_space_size if afterstate else self.action_space_size
        one_hot = torch.zeros(option.shape[0], n, dtype=state.dtype)
        one_hot.scatter_(1, option.long().reshape(-1, 1), 1)
        x = torch.cat((state, one_hot), dim=1)
        if afterstate:
            nxt, reward = self.dynamics_network(x)
            policy_logits, value = self.prediction_network(nxt)
        else:
            nxt, reward = self.afterstate_dynamics_network(x)
            policy_logits, value = self.afterstate_prediction_network(nxt)
        return MZNetworkOutput(value, reward, policy_logits, nxt)


def model_kwargs(name):
    obs, A, C, L, res, hid, sup = CONFIGS[name]
    return dict(observation_shape=obs, action_space_size=A, chance_space_size=C, latent_state_dim=L,
                res_connection_in_dynamics=res, reward_head_hidden_channels=[hid], value_head_hidden_channels=[hid],
                policy_head_hidden_channels=[hid], reward_support_range=sup, value_support_range=sup)


def build(name, seed, dtype=torch.float32):
    torch.manual_seed(seed)
    return emulate_trained_mlp_(StochasticMuZeroModelMLPRef(*CONFIGS[name]), seed).to(dtype).eval()
