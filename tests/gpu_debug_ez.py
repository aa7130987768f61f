"""Warm, back-to-back timings of the EfficientZero per-simulation pieces at the BASELINE config-2 batch (bring-up tool)."""
import os, sys, time
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200 import cabi, ez_tree
from oracle.model_ref import EfficientZeroModelRef, MuZeroModelRef, emulate_trained_

B, A, S = int(os.environ.get("DBG_B", 256)), 6, 50
ez = emulate_trained_(EfficientZeroModelRef((4, 96, 96), A), 0)
mz = emulate_trained_(MuZeroModelRef((4, 96, 96), A), 0)
cez = lzb.EfficientZeroModel(observation_shape=(4, 96, 96), action_space_size=A).load_state_dict(ez.state_dict())
cmz = lzb.MuZeroModel(observation_shape=(4, 96, 96), action_space_size=A).load_state_dict(mz.state_dict())
lat = torch.rand(B, 64, 6, 6).cuda()
act = torch.randint(0, A, (B,)).cuda()
hc = (torch.randn(1, B, 512).cuda() * 0.3, torch.randn(1, B, 512).cuda() * 0.3)


def timeit(fn, n=200):
    for _ in range(20):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n * 1e3


lib = cabi.load()
# raw C-ABI calls with preallocated outputs (no torch allocations inside the timed loop)
nxt = torch.empty(B, 64, 6, 6, device="cuda"); pol = torch.empty(B, A, device="cuda")
rew = torch.empty(B, device="cuda"); val = torch.empty(B, device="cuda")
h0, h1 = hc[0].reshape(B, 512).contiguous(), hc[1].reshape(B, 512).contiguous()
n0, n1 = torch.empty_like(h0), torch.empty_like(h1)
a32 = act.to(torch.int32)
s = cabi.stream_ptr()
t_mz = timeit(lambda: lib.lz_model_recurrent_inference(cmz._h, B, lat.data_ptr(), a32.data_ptr(), nxt.data_ptr(), None, None, pol.data_ptr(), rew.data_ptr(), val.data_ptr(), s))
t_ez = timeit(lambda: lib.lz_model_recurrent_inference_ez(cez._h, B, lat.data_ptr(), h0.data_ptr(), h1.data_ptr(), a32.data_ptr(), nxt.data_ptr(), n0.data_ptr(), n1.data_ptr(), None, None, pol.data_ptr(), rew.data_ptr(), val.data_ptr(), s))
print(f"B={B}: MuZero recurrent (k_net_tc incl. reward FC) {t_mz:.1f} us | EfficientZero recurrent (k_net_tc + LSTM GEMM + head) {t_ez:.1f} us | LSTM+head ~ {t_ez - t_mz:.1f} us")
# tree kernels: traverse + backprop on prepared EZ trees
roots = ez_tree.Roots(B, [list(range(A))] * B)
roots.prepare_no_noise([0.] * B, torch.randn(B, A).cuda(), [-1] * B)
roots._materialize(S, (19652, 1.25, 0.997, 0.01))
t = roots._tree
rs = torch.zeros(B, dtype=torch.int32, device="cuda")
def tree_step():
    lib.lz_tree_traverse(t.h, 0, None, None, t.ix.data_ptr(), t.iy.data_ptr(), t.action.data_ptr(), t.search_len.data_ptr(), t.vtp.data_ptr(), rs.data_ptr(), s)
print(f"tree traverse (EZ, shallow trees): {timeit(tree_step):.1f} us")
