"""The row pitch of the solver's final_scores at the library boundary: mk_solve_pose rejects a pitch below N before it
launches anything, and a caller's layout that the library cannot read in place reaches it as a contiguous copy."""
import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict

pytestmark = pytest.mark.gpu
DEV = "cuda"
GH, GW, B = 15, 14, 2
N = GH * GW


@pytest.fixture(scope="module")
def model():
    cfg = mickey_cfg("vits", 4, 16)
    m = MickeyRelativePose(cfg)
    m.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    m = m.cuda().eval()
    m._engine()._ws_for(B, 14 * GH, 14 * GW)
    return m


def _batch(final_scores):
    g = torch.Generator().manual_seed(0)
    kps = torch.rand(B, 2, N, generator=g) * 200
    depth = torch.rand(B, 1, N, generator=g) + 1
    K = torch.tensor([[[549.7, 0, 268.7], [0, 549.7, 351.8], [0, 0, 1.0]]]).repeat(B, 1, 1)
    b = dict(kps0=kps, kps1=kps.flip(-1), depth_kp0=depth, depth_kp1=depth, K_color0=K, K_color1=K)
    return dict({k: v.to(DEV) for k, v in b.items()}, final_scores=final_scores)


def test_solve_pose_rejects_a_pitch_below_N_before_any_launch(model):
    eng = model._engine()
    b = _batch(torch.rand(B, N, N, device=DEV))
    kps = torch.cat([b["kps0"], b["kps1"]]).contiguous()
    depth = torch.cat([b["depth_kp0"], b["depth_kp1"]]).contiguous()
    pose = torch.empty(B, 13, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    torch.cuda.synchronize()
    launches = eng.launch_count
    p = _lib.ptr
    rc = eng.lib.mk_solve_pose(eng.h, p(b["final_scores"]), N - 1, p(kps), p(depth), p(b["K_color0"]), p(b["K_color1"]), B, N,
                               3, None, None, p(pose), None, None, None, None, p(status), p(eng.ws), eng.ws.numel(),
                               _lib.stream())
    assert rc == -1
    assert b"mk_solve_pose: nn_pitch" in eng.lib.mk_last_error()
    assert eng.launch_count == launches


def test_solve_on_an_expanded_final_scores_equals_its_contiguous_copy(model):
    row = torch.rand(N, generator=torch.Generator().manual_seed(1)).to(DEV)
    fs = row.expand(B, N, N)
    assert fs.stride() == (0, 0, 1)
    poses = []
    for f in (fs, fs.contiguous()):
        b = _batch(f)
        R, t, inl = model.e2e_Procrustes.estimate_pose_vectorized(b, seed=3)
        assert int(b["_solver"]["status"].item()) == 0
        poses.append(torch.cat([R.reshape(B, 9), t.reshape(B, 3), inl], 1))
    assert float(poses[1][:, :9].abs().max()) > 0.5            # a rotation, not the zero pose
    assert torch.equal(poses[0], poses[1])
