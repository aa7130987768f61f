"""The fused ResBlock plans of every supported frame size, as the tower launches them (lz_model_debug_tower_stage).

resblock_tc_plan marks a band down when a conv's tile groups leave one tile on its own: that group would run its 9 taps on a
single accumulator chain per warpgroup.  Here the plans the library actually picked are replayed through the tile grouping of
k_resblock_tc (conv_tc.cu: 6 slabs at 32 channels; at 64 channels 2 slabs in the narrow layout, 4 in the wide one, which a plan
takes once a conv has more than 2 tiles), and no conv may end up in such a group.  A change of the slab counts or of the planner
that brings one back fails here."""
import pytest
import torch

from test_gpu_tower_layers import dump_stage

pytestmark = pytest.mark.gpu

RESBLOCK_STAGES = {1: "resblocks1", 5: "resblocks2", 7: "resblocks3"}


def _slabs(C, NT1, NT2):
    if C == 32:
        return 6
    return 4 if max(NT1, NT2) > 2 else 2


def _groups(NT, MT):
    ng = (NT + MT - 1) // MT
    per = (NT + ng - 1) // ng
    return [min(per, NT - i * per) for i in range(ng)]


@pytest.mark.parametrize("px", [64, 84, 96])
def test_resblock_plans_leave_no_tile_on_its_own(px):
    import lightzero_b200 as lzb
    from lightzero_b200.synthetic_weights import synthetic_state_dict
    cu = lzb.MuZeroModel(observation_shape=(4, px, px), action_space_size=18, downsample=True).load_state_dict(
        synthetic_state_dict((4, px, px), 18))
    obs = torch.zeros(4, 4, px, px, device="cuda")
    for st, name in RESBLOCK_STAGES.items():
        C, H, W, nph, R, G, bh, stages, ctas, npass = dump_stage(cu, obs, st)[1]
        Hin = 2 * H if st == 1 else H                      # resblocks1 writes the phase split of its 2H-row output
        pitch = Hin + 1
        S = (bh + 4) * pitch + 2
        NT1 = ((G - 1) * S + (bh + 2) * pitch + 127) // 128
        NT2 = ((G - 1) * S + bh * pitch + 127) // 128
        MT = _slabs(C, NT1, NT2)
        for conv, NT in (("conv1", NT1), ("conv2", NT2)):
            g = _groups(NT, MT)
            assert not (NT > 1 and 1 in g), f"{px} px {name} {conv}: {NT} tiles run as groups {g} (G = {G}, band_h = {bh})"
