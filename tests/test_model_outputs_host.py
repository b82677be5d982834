"""CPU tests of the model's output plumbing, on hand-built solver outputs: the inlier list that the staged solver,
forward() and pose_from_features() share, the data-dict fill and the views of the pose rows."""
import pytest
import torch

from mickey_b200.model import _inlier_list, _pose_views, _set_correspondences

B, GRID, S, IM = 2, (2, 3), 5, 3
N = GRID[0] * GRID[1]


def _solver_case(status=0):
    """Two pairs, S = 5 sampled cells per set, IM = 3 sets per pair.  The winning sets (rows 1 and 5) hold distinct cells;
    every cell outside their inlier masks scores 2, above every masked one, so any unmasked row would sort first."""
    g = torch.Generator().manual_seed(0)
    kps0, kps1 = torch.rand(B, 2, N, generator=g) * 500, torch.rand(B, 2, N, generator=g) * 500
    depth0, depth1 = torch.rand(B, 1, N, generator=g) * 10, torch.rand(B, 1, N, generator=g) * 10
    final = torch.full((B, N, N + 2), 2.0)[:, :, :N]                  # a padded-pitch view, as the engine hands out
    sampled = torch.randint(0, N * N, (B * IM, S), generator=g, dtype=torch.int32)
    sampled[1] = torch.tensor([7, 0, 35, 14, 20])
    sampled[5] = torch.tensor([3, 33, 12, 28, 9])
    best_set = torch.tensor([1, 5], dtype=torch.int32)
    mask = torch.tensor([[1.0, 0.0, 1.0, 1.0, 0.0], [0.0, 1.0, 1.0, 1.0, 1.0]])
    for b in range(B):
        for s in range(S):
            if mask[b, s] > 0.5:
                i, j = divmod(int(sampled[best_set[b], s]), N)
                final[b, i, j] = torch.rand((), generator=g)
    solver = {"best_set": best_set, "sampled_idx": sampled, "inlier_mask": mask, "status": torch.tensor([status], dtype=torch.int32)}
    return solver, final, kps0, kps1, depth0, depth1


def test_inlier_rows_are_the_masked_cells_by_descending_score():
    solver, final, kps0, kps1, depth0, depth1 = _solver_case()
    got = _inlier_list(solver, final, kps0, kps1, depth0, depth1)
    assert len(got) == B
    for b in range(B):
        want = []
        for s in range(S):
            if solver["inlier_mask"][b, s] > 0.5:
                i, j = divmod(int(solver["sampled_idx"][solver["best_set"][b], s]), N)
                want.append([float(v) for v in (kps0[b, 0, i], kps0[b, 1, i], kps1[b, 0, j], kps1[b, 1, j], final[b, i, j],
                                                depth0[b, 0, i], depth1[b, 0, j])])
        want.sort(key=lambda r: -r[4])
        assert got[b].shape == (int(solver["inlier_mask"][b].sum()), 7)
        assert torch.equal(got[b], torch.tensor(want))
        assert bool((got[b][:, 4] < 1).all())                        # no unmasked cell (score 2) made it in
        assert bool((got[b][1:, 4] < got[b][:-1, 4]).all())


@pytest.mark.parametrize("bit", [0, 1, 2, 3])
def test_each_zero_pose_status_bit_empties_every_pair(bit):
    got = _inlier_list(*_solver_case(status=1 << bit))
    assert len(got) == B
    for t in got:
        assert t.shape == (0, 5) and t.dtype == torch.float32 and t.device.type == "cpu"


@pytest.mark.parametrize("lean", [False, True])
def test_correspondence_keys_are_views_of_the_given_tensors(lean):
    n, (gh, gw) = B, GRID
    kps, depth = torch.rand(2 * n, 2, N), torch.rand(2 * n, 1, N)
    scr, dsc = (torch.rand(n, 1, N), torch.rand(n, 1, N)), (torch.rand(n, 128, N), torch.rand(n, 128, N))
    scores = None if lean else torch.rand(n, N, N)
    kp_scores = None if lean else torch.rand(n, N, N)
    data = {"image0": None}
    _set_correspondences(data, kps, depth, scr, dsc, GRID, 14, scores, kp_scores)
    assert data["kps0_shape"] == data["kps1_shape"] == [gh, gw] and data["down_factor"] == 14
    assert torch.equal(data["kps0"], kps[:n]) and torch.equal(data["kps1"], kps[n:])
    assert torch.equal(data["depth_kp0"], depth[:n]) and torch.equal(data["depth_kp1"], depth[n:])
    assert torch.equal(data["depth0_map"], depth[:n].reshape(n, 1, gh, gw))
    assert torch.equal(data["depth1_map"], depth[n:].reshape(n, 1, gh, gw))
    assert data["scr0"] is scr[0] and data["scr1"] is scr[1] and data["dsc0"] is dsc[0] and data["dsc1"] is dsc[1]
    for k in ("kps0", "kps1", "depth_kp0", "depth_kp1", "depth0_map", "depth1_map"):
        assert data[k].untyped_storage().data_ptr() == (kps if k.startswith("kps") else depth).untyped_storage().data_ptr(), k
    if lean:
        assert "scores" not in data and "kp_scores" not in data
    else:
        assert data["scores"] is scores and data["kp_scores"] is kp_scores
    assert "image0" in data


def test_pose_views_split_the_pose_rows_without_copies():
    pose = torch.arange(3 * 13, dtype=torch.float32).reshape(3, 13)
    R, t, inliers = _pose_views(pose)
    assert R.shape == (3, 3, 3) and t.shape == (3, 1, 3) and inliers.shape == (3, 1)
    for b in range(3):
        assert torch.equal(R[b], pose[b, :9].reshape(3, 3))
        assert torch.equal(t[b, 0], pose[b, 9:12]) and inliers[b, 0] == pose[b, 12]
    for v in (R, t, inliers):
        assert v.untyped_storage().data_ptr() == pose.untyped_storage().data_ptr()
