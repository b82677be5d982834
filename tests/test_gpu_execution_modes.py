"""The execution modes bench.py times, byte for byte against the staged path.

Every fp64 check of the kernel stages runs on the staged path: mk_extract + mk_match + mk_solve_pose launched eagerly on
the caller's stream at pipeline depth 1.  bench.py times other paths of the same computation: mk_forward replayed from
CUDA graphs, three engines on side streams (pipeline_depth = 3) with assume_inputs_ready and static_outputs, pinned host
images next to device K.  None of them may change a bit: there are no float atomics, and every path draws the solver
seed from the torch RNG at the same point.  So each mode here runs a sequence of steps, every step with its own images
and its own K, and every output of every step must be torch.equal to the staged path's output for that step.

Ordering defects show up as wrong values only when the timing lines up; the input operands (images, K) are therefore
produced on the caller's stream behind a spin kernel (torch.cuda._sleep, ~20 ms), so that a missing wait reads stale
values every time.  Workspace lifetimes and the ordering of handle calls are checked structurally instead: which
stream owns each engine buffer, and whether a bank call can complete before engine 0's stream does.
"""
import os
import subprocess
import sys

import pytest
import torch

from mickey_b200 import _lib
from mickey_b200.config import mickey_cfg
from mickey_b200.model import MickeyRelativePose
from mickey_b200.weights import synthetic_state_dict
from tests.common import K_TOY, ROOT

pytestmark = pytest.mark.gpu
DEV = "cuda"
SPIN = 40_000_000           # cycles of torch.cuda._sleep: ~20-25 ms at the H100's 1.6-2.0 GHz, far below 0.2 s
S_SMALL, T_SMALL = (210, 196), (224, 182)
KEYS = ("R", "t", "inliers", "kps0", "kps1", "depth_kp0", "depth_kp1", "depth0_map", "depth1_map", "scr0", "scr1",
        "dsc0", "dsc1", "scores", "kp_scores", "final_scores")
LEAN_DROPS = ("scores", "kp_scores")


# ---------------------------------------------------------------------------------------------------------------
# inputs, models, the staged reference
# ---------------------------------------------------------------------------------------------------------------
def step_inputs(k, B, H, W, u8=False):
    """Host inputs of step k: its own images and its own K (per pair), fp32 [B,3,H,W] or uint8 [B,H,W,3]."""
    g = torch.Generator().manual_seed(1000 + k)
    if u8:
        im0 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
        im1 = torch.randint(0, 256, (B, H, W, 3), generator=g, dtype=torch.uint8)
    else:
        im0, im1 = torch.rand(B, 3, H, W, generator=g), torch.rand(B, 3, H, W, generator=g)
    K = torch.tensor(K_TOY).repeat(B, 1, 1)
    scale = 1.0 + 0.02 * (k % 7) + 0.005 * torch.arange(B).view(B, 1, 1)
    K0 = K.clone()
    K0[:, :2, :] *= scale
    K1 = K.clone()
    K1[:, 0, 2] += 3.0 * (k + 1)
    K1[:, 1, 2] -= 2.0 * (k + 1)
    return {"image0": im0, "image1": im1, "K_color0": K0, "K_color1": K1}


def make_model(variant, im, ir, wseed=0, sd=None):
    cfg = mickey_cfg(variant, im, ir)
    m = MickeyRelativePose(cfg)
    m.load_state_dict(sd if sd is not None else synthetic_state_dict(cfg, seed=wseed), strict=True)
    return m.cuda().eval()


def seed_of(k):
    return 7000 + k


def collect(data, return_inliers=False):
    out = {k: data[k].clone() for k in KEYS if k in data}
    if return_inliers:
        out["inliers_list"] = [x.clone() for x in data["inliers_list"]]
    return out


def staged_step(model, host, k, return_inliers=False):
    """The reference: the staged path, eager, depth 1, on device copies of the host inputs."""
    model.staged, model.pipeline_depth = True, 1
    data = {n: v.to(DEV) for n, v in host.items()}
    torch.manual_seed(seed_of(k))
    model(data, return_inliers=return_inliers)
    out = collect(data, return_inliers)
    torch.cuda.synchronize()
    model.staged = False
    return out


def assert_equal_outputs(got, ref, what, skip=()):
    for name in KEYS:
        if name in skip:
            assert name not in got, (what, name)
            continue
        assert name in got, (what, name)
        a, b = got[name], ref[name]
        assert a.shape == b.shape and torch.equal(a, b), \
            f"{what}: {name} differs ({int((a != b).sum()) if a.shape == b.shape else 'shape'} elements)"
    if "inliers_list" in got:
        assert len(got["inliers_list"]) == len(ref["inliers_list"])
        for b, (x, y) in enumerate(zip(got["inliers_list"], ref["inliers_list"])):
            assert x.shape == y.shape and torch.equal(x.cpu(), y.cpu()), f"{what}: inliers_list[{b}] differs"


def assert_steps_distinguishable(refs):
    """The harness can fail: every output of step k differs from step k-1's, so a step that read a neighbouring step's
    buffers cannot pass."""
    for k in range(1, len(refs)):
        a, b = refs[k], refs[k - 1]
        for name in KEYS:
            if name in a and name in b and a[name].shape == b[name].shape:
                assert not torch.equal(a[name], b[name]), f"steps {k - 1} and {k} give the same {name}"


def spin_then_device(host, fp64_k=False, spin=True):
    """Device copies of the host inputs produced on the current stream behind a spin kernel: until the spin ends,
    the device tensors hold whatever their blocks held before."""
    dev = {n: torch.empty(v.shape, dtype=torch.float64 if (fp64_k and n.startswith("K")) else v.dtype, device=DEV)
           for n, v in host.items()}
    if spin:
        torch.cuda._sleep(SPIN)
    for n, v in host.items():
        dev[n].copy_(v.pin_memory(), non_blocking=True)
    return dev


class Refs:
    """Staged references of the steps of one model configuration, computed once per (B, H, W, u8, k)."""

    def __init__(self, variant="vits", im=2, ir=8, wseed=0, sd=None):
        self.model = make_model(variant, im, ir, wseed, sd)
        self.cache = {}

    def __call__(self, k, B, H, W, u8=False, return_inliers=False):
        key = (k, B, H, W, u8, return_inliers)
        if key not in self.cache:
            self.cache[key] = staged_step(self.model, step_inputs(k, B, H, W, u8), k, return_inliers)
        return self.cache[key]


@pytest.fixture(scope="module")
def refs_s():
    return Refs("vits", 2, 8, 0)


def run_step(model, data, k, return_inliers=False):
    torch.manual_seed(seed_of(k))
    model(data, return_inliers=return_inliers)
    return collect(data, return_inliers)


# ---------------------------------------------------------------------------------------------------------------
def test_eager_forward_equals_staged(refs_s):
    """mk_forward (one C call, eager) gives the staged path's bytes: the fp64 checks of the stages carry over."""
    model = make_model("vits", 2, 8, 0)
    model.use_graph = False
    for k in range(3):
        for (H, W), B in ((S_SMALL, 2), (T_SMALL, 1)):
            data = {n: v.to(DEV) for n, v in step_inputs(k, B, H, W).items()}
            got = run_step(model, data, k, return_inliers=True)
            torch.cuda.synchronize()
            assert_equal_outputs(got, refs_s(k, B, H, W, return_inliers=True), f"eager step {k} {H}x{W}")


def test_graph_depth1_distinct_steps(refs_s):
    """Eager call, capture and replay on both buffer sets, each step with its own inputs."""
    model = make_model("vits", 2, 8, 0)
    refs = [refs_s(k, 2, *S_SMALL) for k in range(7)]
    assert_steps_distinguishable(refs)
    outs = []
    for k in range(7):
        data = spin_then_device(step_inputs(k, 2, *S_SMALL))
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    eng = model._engine()
    assert all(eng._graphs[(2, *S_SMALL, s, (False, False))]["graph"] is not None for s in (0, 1))
    for k, (o, r) in enumerate(zip(outs, refs)):
        assert_equal_outputs(o, r, f"graph step {k}")


@pytest.mark.parametrize("depth", [2, 3])
def test_pipelined_device_inputs_wait_for_the_caller(refs_s, depth):
    """pipeline_depth 2 / 3 with device inputs produced behind a spin kernel: each engine's stream waits on the caller's."""
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = depth
    n = 4 * depth + 1
    outs = []
    for k in range(n):
        data = spin_then_device(step_inputs(k, 1, *T_SMALL))
        outs.append(run_step(model, data, k, return_inliers=(k % 3 == 0)))
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *T_SMALL, return_inliers=(k % 3 == 0)), f"depth {depth} step {k}")


def test_throughput_mode_static_outputs_valid_for_their_window(refs_s):
    """bench.py's throughput mode: depth 3, assume_inputs_ready, static_outputs.  Outputs are read right after each call
    and, for every fourth call, again 2*depth - 1 calls later: the end of the window in which Engine.forward says they
    stay valid.  Under assume_inputs_ready that window holds in host order, so the test keeps the contract: the reads
    of call k - 2*depth have completed before call k is issued (one event per call, 2*depth calls back)."""
    depth, n = 3, 16
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth, model.assume_inputs_ready, model.static_outputs = depth, True, True
    inputs = [{n_: v.to(DEV) for n_, v in step_inputs(k, 1, *S_SMALL).items()} for k in range(n)]
    torch.cuda.synchronize()                          # the inputs are ready, as the mode assumes
    views, first, late, read = [], [], {}, {}
    for k in range(n):
        if k >= 2 * depth:
            read.pop(k - 2 * depth).synchronize()     # call k reuses call k - 2*depth's buffer set
        data = dict(inputs[k])
        torch.manual_seed(seed_of(k))
        model(data)
        views.append({name: data[name] for name in KEYS})
        first.append({name: v.clone() for name, v in views[-1].items()})
        read[k] = torch.cuda.Event()
        read[k].record()
        j = k - (2 * depth - 1)
        if j >= 0 and j % 4 == 1:
            late[j] = {name: v.clone() for name, v in views[j].items()}
            read[j].record()
    torch.cuda.synchronize()
    assert len(late) >= 3
    for k in range(n):
        ref = refs_s(k, 1, *S_SMALL)
        assert_equal_outputs(first[k], ref, f"static step {k} read at once")
        if k in late:
            assert_equal_outputs(late[k], ref, f"static step {k} read {2 * depth - 1} calls later")


def test_released_outputs_order_the_next_use_of_their_buffer_set(refs_s):
    """The default (cloning) forward under assume_inputs_ready at depth 2: the engine does not wait on the caller's
    stream, yet the call that reuses a buffer set must run after the caller's reads (clones) of that set's previous
    outputs.  With the caller's stream held by a spin kernel in front of call j's clones, call j + 4 (same engine, same
    buffer set) must not complete before the spin does."""
    depth = 2
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth, model.assume_inputs_ready = depth, True
    inputs = [{n_: v.to(DEV) for n_, v in step_inputs(k, 1, *S_SMALL).items()} for k in range(10)]
    torch.cuda.synchronize()
    outs = []
    for k in range(10):
        if k == 6:
            torch.cuda._sleep(SPIN)                   # call 6's clones (and its release) queue behind this
            held = torch.cuda.Event()
            held.record()
        outs.append(run_step(model, dict(inputs[k]), k))
        if k == 6 + 2 * depth:
            eng = model._engine_pool()[k % depth]
            after = torch.cuda.Event()
            after.record(eng.stream)
            after.synchronize()
            assert held.query(), "the buffer set was reused before the caller's reads of its previous outputs"
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL), f"released step {k}")


@pytest.mark.parametrize("k_where", ["host", "device", "device64"])
@pytest.mark.parametrize("depth", [1, 2])
@pytest.mark.parametrize("u8", [False, True], ids=["fp32", "uint8"])
def test_pinned_host_images_with_host_and_device_k(refs_s, depth, u8, k_where):
    """Pinned host images (the engine's copy stream) next to K on the host, K on the device behind a spin kernel, or
    fp64 K on the device behind a spin kernel (converted to fp32 by the engine)."""
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = depth
    outs = []
    for k in range(5):
        host = step_inputs(k, 1, *S_SMALL, u8=u8)
        data = {"image0": host["image0"].pin_memory(), "image1": host["image1"].pin_memory()}
        if k_where == "host":
            data.update(K_color0=host["K_color0"], K_color1=host["K_color1"])
        else:
            data.update(spin_then_device({"K_color0": host["K_color0"], "K_color1": host["K_color1"]},
                                         fp64_k=(k_where == "device64")))
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL, u8=u8), f"host images, K {k_where}, depth {depth}, step {k}")


@pytest.mark.parametrize("depth", [1, 2])
def test_new_buffer_sets_wait_for_the_caller(refs_s, depth):
    """A new buffer set takes its blocks on the caller's stream, where kernels of the tensors that held them before may
    still be queued, so the copy stream writes host images into it only behind the caller's stream.  With the caller's
    stream held by a spin kernel that produces K, the copy stream's work for each new buffer set must not complete
    before the spin."""
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = depth
    outs = []
    for k in range(2 * depth):                  # every engine's two buffer sets, each new
        host = step_inputs(k, 1, *S_SMALL)
        eng = model._engine_pool()[model.__dict__.get("_turn", 0) % depth]
        data = {"image0": host["image0"].pin_memory(), "image1": host["image1"].pin_memory()}
        data.update(spin_then_device({"K_color0": host["K_color0"], "K_color1": host["K_color1"]}))
        held = torch.cuda.Event()
        held.record()
        outs.append(run_step(model, data, k))
        copied = torch.cuda.Event()
        copied.record(eng._copy_stream)
        copied.synchronize()
        assert held.query(), f"step {k}: host images were copied into a new buffer set ahead of the caller's stream"
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL), f"new buffer set, depth {depth}, step {k}")


def test_lean_outputs_on_their_own_buffer_sets(refs_s):
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = 2
    outs = []
    for k in range(10):
        model.lean_outputs = k % 5 >= 2                 # full, full, lean, lean, lean, ...: both kinds of graph per engine
        data = spin_then_device(step_inputs(k, 1, *S_SMALL))
        outs.append((model.lean_outputs, run_step(model, data, k, return_inliers=True)))
    torch.cuda.synchronize()
    for k, (lean, o) in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL, return_inliers=True), f"lean={lean} step {k}",
                             skip=LEAN_DROPS if lean else ())


def test_batch_growth_while_other_steps_are_in_flight(refs_s):
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = 2
    sizes = [2, 3, 1, 3, 2, 3, 1, 3]
    outs = []
    for k, B in enumerate(sizes):
        data = spin_then_device(step_inputs(k, B, *S_SMALL))
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    for k, (B, o) in enumerate(zip(sizes, outs)):
        assert_equal_outputs(o, refs_s(k, B, *S_SMALL), f"B={B} step {k}")


GEOMS = [S_SMALL, T_SMALL, (196, 196), (182, 224), (168, 210)]


def test_five_geometries_evict_and_recapture(refs_s):
    """MAX_GEOMETRIES = 4: the fifth geometry evicts the first one; going back to it rebuilds its tables and graphs."""
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = 2
    seq = [g for g in GEOMS for _ in range(6)] + [GEOMS[0]] * 8 + [GEOMS[1]] * 2
    outs = []
    for k, (H, W) in enumerate(seq):
        data = spin_then_device(step_inputs(k, 1, H, W))
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    assert all(len(e._geo_state) <= e.MAX_GEOMETRIES for e in model._engine_pool())
    for k, ((H, W), o) in enumerate(zip(seq, outs)):
        assert_equal_outputs(o, refs_s(k, 1, H, W), f"{H}x{W} step {k}")


def test_weight_reload_between_pipelined_steps(refs_s):
    cfg = mickey_cfg("vits", 2, 8)
    sd_b = synthetic_state_dict(cfg, seed=5)
    refs_b = Refs(sd=sd_b)
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = 2
    plan = [("a", k) for k in range(5)] + [("b", k) for k in range(5, 10)] + [("a", k) for k in range(10, 13)]
    outs, cur = [], "a"
    for which, k in plan:
        if which != cur:
            model.load_state_dict(sd_b if which == "b" else synthetic_state_dict(cfg, seed=0), strict=True)
            cur = which
        data = spin_then_device(step_inputs(k, 1, *S_SMALL))
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    for (which, k), o in zip(plan, outs):
        ref = (refs_s if which == "a" else refs_b)(k, 1, *S_SMALL)
        assert_equal_outputs(o, ref, f"weights {which} step {k}")
    assert not torch.equal(refs_b(6, 1, *S_SMALL)["dsc0"], refs_s(6, 1, *S_SMALL)["dsc0"])


def test_depth_changes_as_bench_toggles_them(refs_s):
    """depth 1 -> 3 -> 1 in one sequence, with assume_inputs_ready switched on for depth 3 and off again (bench.measure):
    engine 0 gains a side stream after its graphs were captured on the caller's stream."""
    model = make_model("vits", 2, 8, 0)
    outs, k = [], 0
    for depth, assume, n in ((1, False, 5), (3, True, 13), (1, False, 5)):
        model.pipeline_depth, model.assume_inputs_ready = depth, assume
        if assume:
            block = [{n_: v.to(DEV) for n_, v in step_inputs(k + i, 1, *S_SMALL).items()} for i in range(n)]
            torch.cuda.synchronize()                  # ready before the block, as the mode assumes
        else:
            block = [None] * n
        for i in range(n):
            data = dict(block[i]) if assume else spin_then_device(step_inputs(k, 1, *S_SMALL))
            outs.append((depth, k, run_step(model, data, k)))
            k += 1
    torch.cuda.synchronize()
    for depth, k, o in outs:
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL), f"depth {depth} step {k}")


def test_bank_calls_between_pipelined_steps(refs_s):
    """extract_features / pose_from_features on engine 0's handle while forward steps are in flight at depth 2: every
    bank result equals the same call made alone, the forward steps still equal the reference, and a bank call does not
    complete before the work queued on engine 0's stream."""
    model = make_model("vits", 2, 8, 0)
    model.pipeline_depth = 2
    alone = make_model("vits", 2, 8, 0)
    imgs = torch.rand(4, 3, *S_SMALL, generator=torch.Generator().manual_seed(77))
    K = torch.tensor(K_TOY).repeat(2, 1, 1)

    def bank_calls(m, s):
        feats = m.extract_features(imgs.to(DEV))
        torch.manual_seed(s)
        d = m.pose_from_features(feats, [0, 2], feats, [1, 3], K, K, return_inliers=True)
        return [t.clone() for t in feats.tensors()], {n: (v.clone() if torch.is_tensor(v) else v) for n, v in d.items()}

    outs, banks = [], []
    for k in range(10):
        data = spin_then_device(step_inputs(k, 1, *S_SMALL))
        outs.append(run_step(model, data, k))
        if k % 3 == 2:
            eng0 = model._engine()
            assert eng0.stream is not None
            with torch.cuda.stream(eng0.stream):
                torch.cuda._sleep(SPIN)
                held = torch.cuda.Event()
                held.record()
            banks.append((k, bank_calls(model, 900 + k)))
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
            assert held.query(), "a bank call completed before the work queued on engine 0's stream"
    torch.cuda.synchronize()
    for k, o in enumerate(outs):
        assert_equal_outputs(o, refs_s(k, 1, *S_SMALL), f"forward step {k} between bank calls")
    for k, (feats, d) in banks:
        feats_a, d_a = bank_calls(alone, 900 + k)
        for x, y in zip(feats, feats_a):
            assert torch.equal(x, y), f"bank features after step {k}"
        for n in KEYS:
            assert torch.equal(d[n], d_a[n]), f"pose_from_features {n} after step {k}"
        for x, y in zip(d["inliers_list"], d_a["inliers_list"]):
            assert torch.equal(x.cpu(), y.cpu())


def test_engine_buffers_belong_to_their_streams(refs_s, monkeypatch):
    """Every engine buffer belongs to (was allocated on) the stream that uses it, or was passed to record_stream for it,
    after a sequence that grows batches, evicts a geometry, reloads weights and changes the depth."""
    recorded = set()
    orig = torch.Tensor.record_stream

    def spy(self, stream):
        recorded.add((self.untyped_storage().data_ptr(), stream.cuda_stream))
        return orig(self, stream)

    monkeypatch.setattr(torch.Tensor, "record_stream", spy)
    cfg = mickey_cfg("vits", 2, 8)
    model = make_model("vits", 2, 8, 0)
    k = 0
    for depth, B, geo in ((1, 1, S_SMALL), (1, 2, S_SMALL), (2, 1, S_SMALL), (2, 3, S_SMALL), (3, 1, T_SMALL),
                          (2, 1, GEOMS[2]), (2, 1, GEOMS[3]), (2, 1, GEOMS[4]), (2, 2, S_SMALL)):
        model.pipeline_depth = depth
        for _ in range(2 * depth + 1):
            data = {n: v.to(DEV) for n, v in step_inputs(k, B, *geo).items()}
            data["image0"] = data["image0"].cpu().pin_memory() if k % 2 else data["image0"]
            data["image1"] = data["image1"].cpu().pin_memory() if k % 2 else data["image1"]
            run_step(model, data, k)
            k += 1
        if depth == 2 and B == 3:
            model.load_state_dict(synthetic_state_dict(cfg, seed=0), strict=True)
    torch.cuda.synchronize()
    segs = [(s["address"], s["address"] + s["total_size"], s["stream"]) for s in torch.cuda.memory_snapshot()]
    caller = torch.cuda.current_stream().cuda_stream

    def owner(ptr):
        hit = [s for s in segs if s[0] <= ptr < s[1]]
        assert len(hit) == 1, hex(ptr)
        return hit[0][2]

    engines = model._engine_pool()
    assert len(engines) == 2 and all(e.stream is not None for e in engines)
    checked = 0
    for e in engines:
        users = {e.stream.cuda_stream}
        for t in e._buffers():
            if t is None:
                continue
            p = t.untyped_storage().data_ptr()
            for s in users:
                assert owner(p) == s or (p, s) in recorded, f"engine buffer {hex(p)} is used on stream {s:#x} unrecorded"
            checked += 1
        for ent in e._graphs.values():                  # the outputs are read on the caller's stream
            for t in ent["st"].values():
                if t is not None:
                    p = t.untyped_storage().data_ptr()
                    assert owner(p) == caller or (p, caller) in recorded
    assert checked > 20


# ---------------------------------------------------------------------------------------------------------------
def test_bench_c2_sequence_with_outputs_checked():
    """bench.measure at C2 (ViT-S, 8 x 64, one 720x540 pair, static outputs): depth-1 steps, depth-3 steps with
    assume_inputs_ready, pinned-host steps with device K, then depth 1 again; every step checked against the staged path."""
    H, W = 720, 540
    ref_model = make_model("vits", 8, 64, 0)
    model = make_model("vits", 8, 64, 0)
    model.static_outputs = True
    plan = [(1, False, "dev")] * 3 + [(3, True, "dev")] * 12 + [(3, True, "host")] * 9 + [(1, False, "dev")] * 2
    ready = [{n: v.to(DEV) for n, v in step_inputs(k, 1, H, W).items()} for k in range(len(plan))]
    pinned = [{"image0": step_inputs(k, 1, H, W)["image0"].pin_memory(),
               "image1": step_inputs(k, 1, H, W)["image1"].pin_memory()} for k in range(len(plan))]
    torch.cuda.synchronize()
    outs = []
    for k, (depth, assume, src) in enumerate(plan):
        model.pipeline_depth, model.assume_inputs_ready = depth, assume
        data = dict(ready[k])
        if src == "host":
            data.update(pinned[k])
        outs.append(run_step(model, data, k))
    torch.cuda.synchronize()
    refs = []
    for k in range(len(plan)):
        refs.append(staged_step(ref_model, step_inputs(k, 1, H, W), k))
        assert_equal_outputs(outs[k], refs[k], f"C2 step {k} {plan[k]}")
        if k:
            assert_steps_distinguishable(refs[-2:])
            refs[-2] = None


# ---------------------------------------------------------------------------------------------------------------
PDL_CASES = (("vits", 2, 8, 0, 2, S_SMALL), ("vitb", 2, 8, 1, 1, T_SMALL))


def pdl_outputs(path=None):
    """The steps compared with and without programmatic dependent launch: one ViT-S and one small ViT-B batch, eager and
    from graphs.  Writes the outputs to `path` (the subprocess) or returns them."""
    res = {"pdl": bool(_lib.load().mk_pdl_enabled())}
    for variant, im, ir, wseed, B, (H, W) in PDL_CASES:
        model = make_model(variant, im, ir, wseed)
        for k in range(4):
            data = {n: v.to(DEV) for n, v in step_inputs(k, B, H, W).items()}
            res[f"{variant}/{k}"] = {n: v.cpu() for n, v in run_step(model, data, k).items()}
    torch.cuda.synchronize()
    if path is None:
        return res
    torch.save(res, path)


def test_pdl_off_gives_the_same_bytes(tmp_path):
    assert os.environ.get("MICKEY_PDL", "1") != "0", "this process must run with PDL on"
    path = tmp_path / "pdl_off.pt"
    env = dict(os.environ, MICKEY_PDL="0", MICKEY_SYNTHETIC_BACKBONE="1")
    code = ("import sys; sys.path.insert(0, sys.argv[1]); from tests.test_gpu_execution_modes import pdl_outputs; "
            "pdl_outputs(sys.argv[2])")
    py = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    r = subprocess.run(py + ["-c", code, ROOT, str(path)], env=env, cwd=ROOT, timeout=240,
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    off = torch.load(path)
    on = pdl_outputs()
    assert on["pdl"] and not off["pdl"]
    for variant, *_ in PDL_CASES:
        for k in range(4):
            a, b = on[f"{variant}/{k}"], off[f"{variant}/{k}"]
            assert set(a) == set(b)
            for n in a:
                assert torch.equal(a[n], b[n]), f"{variant} step {k}: {n} differs with MICKEY_PDL=0"
