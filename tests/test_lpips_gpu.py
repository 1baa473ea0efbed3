"""GPU tests of evaluation.lpips against the fp64 restatement (tests/lpips_reference.py): accuracy of every frame's score
and every tap score on structured frames (smooth fields plus noise, renders at several perturbation sizes and unrelated
images) at sizes from the smallest frame to 1008 x 756 and 37 frames; the default and explicit masks; and the exact
properties: a frame against itself scores 0, the score is symmetric, a frame's score does not depend on its batch or
workspace chunk, reruns and CUDA-graph replays are bit-identical."""
import numpy as np
import pytest
import torch

from tests import lpips_reference as R

pytestmark = pytest.mark.gpu

TOL = 5e-4   # absolute, on the score and on every tap score: the third decimal LPIPS is reported to


@pytest.fixture(scope="module")
def setup():
    from nonrigid_nerf_b200 import evaluation as E
    sd = R.random_state_dict(0)
    return E, sd, E.lpips_weights(sd)


def _cuda(*a):
    return [torch.from_numpy(x).cuda() for x in a]


@pytest.mark.parametrize("f,h,w", [(1, 31, 31), (1, 37, 53), (3, 378, 504), (1, 756, 1008), (37, 378, 504)])
def test_accuracy_against_fp64(setup, f, h, w):
    E, sd, wt = setup
    gt, gen = R.frames(10 + f + h, f, h, w)
    if f == 1:   # a single frame: an unrelated render and a perturbed one would otherwise not both appear
        gt2, gen2 = R.frames(11 + h, 6, h, w)
        gt, gen = np.concatenate([gt, gt2[5:]]), np.concatenate([gen, gen2[5:]])
    ref, ref_per = R.lpips(gt, gen, sd)
    g, r = _cuda(gt, gen)
    out, per = E.lpips(g, r, wt, per_layer=True)
    torch.cuda.synchronize()
    out, per = out.cpu().double().numpy(), per.cpu().double().numpy()
    err, err_per = np.abs(out - ref).max(), np.abs(per - ref_per).max(axis=0)
    print(f"\n{f}x{h}x{w}: LPIPS {np.round(ref, 4).tolist()[:8]} max |err| {err:.2e}, per tap {np.array2string(err_per, precision=2)}")
    assert err <= TOL and err_per.max() <= TOL, (err, err_per)
    assert out[0] == 0.0 and np.all(per[0] == 0.0)   # frame 0's render is its ground truth
    assert torch.equal(E.lpips(g, r, wt).cpu(), torch.from_numpy(out).float())   # per_layer does not change the score


def test_default_and_explicit_mask(setup):
    E, sd, wt = setup
    gt, gen = R.frames(21, 4, 64, 80)
    gt[0, 5:20, 10:30] = 0   # the default mask: pixels of gt[0] whose channels sum to 0
    ref, ref_per = R.lpips(gt, gen, sd)
    g, r = _cuda(gt, gen)
    out, per = E.lpips(g, r, wt, per_layer=True)
    assert np.abs(out.cpu().numpy() - ref).max() <= TOL and np.abs(per.cpu().numpy() - ref_per).max() <= TOL
    explicit = np.zeros((64, 80), dtype=bool)
    explicit[30:50, 40:79] = True
    ref2, _ = R.lpips(gt, gen, sd, mask=explicit)
    out2 = E.lpips(g, r, wt, mask=torch.from_numpy(explicit).cuda())
    assert np.abs(out2.cpu().numpy() - ref2).max() <= TOL
    assert np.abs(ref2 - ref).max() > 10 * TOL   # the two masks give different scores
    # the default equals the same mask given explicitly, bit for bit
    assert torch.equal(out, E.lpips(g, r, wt, mask=torch.from_numpy(R.mask_from(gt[0])).cuda()))


def test_exact_properties(setup):
    E, sd, wt = setup
    f, h, w = 37, 378, 504
    gt, gen = R.frames(33, f, h, w)
    g, r = _cuda(gt, gen)
    one = torch.zeros((h, w), dtype=torch.uint8, device="cuda")   # explicit mask: frames scored alone use the same one
    out, per = E.lpips(g, r, wt, mask=one, per_layer=True)
    self_score, self_per = E.lpips(g, g, wt, mask=one, per_layer=True)
    assert torch.all(self_score == 0) and torch.all(self_per == 0)
    back, back_per = E.lpips(r, g, wt, mask=one, per_layer=True)
    assert torch.equal(back, out) and torch.equal(back_per, per)
    # chunks of 18, 18 and 1 by default; of 5 and of 1 here; and every frame alone
    for chunk in (5, 1):
        o, p = E.lpips(g, r, wt, mask=one, per_layer=True, chunk_frames=chunk)
        assert torch.equal(o, out) and torch.equal(p, per), chunk
    for i in (0, 4, 17, 18, 36):
        o, p = E.lpips(g[i:i + 1], r[i:i + 1], wt, mask=one, per_layer=True)
        assert torch.equal(o[0], out[i]) and torch.equal(p[0], per[i]), i
    again, again_per = E.lpips(g, r, wt, mask=one, per_layer=True)
    assert torch.equal(again, out) and torch.equal(again_per, per)


def test_graph_replay_equals_eager(setup):
    E, sd, wt = setup
    gt, gen = R.frames(44, 5, 96, 128)
    g, r = _cuda(gt, gen)
    eager, eager_per = E.lpips(g, r, wt, per_layer=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        E.lpips(g, r, wt, per_layer=True)   # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, per = E.lpips(g, r, wt, per_layer=True)
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and torch.equal(per, eager_per)


def test_empty_batch_and_refusals(setup):
    E, sd, wt = setup
    x = torch.zeros((0, 40, 40, 3), device="cuda")
    out, per = E.lpips(x, x, wt, per_layer=True)
    assert out.shape == (0,) and per.shape == (0, 5)
    small = torch.zeros((1, 30, 64, 3), device="cuda")
    with pytest.raises(RuntimeError, match="at least 31"):
        E.lpips(small, small, wt)
    with pytest.raises(RuntimeError, match="differ"):
        E.lpips(torch.zeros((1, 40, 40, 3), device="cuda"), torch.zeros((1, 40, 41, 3), device="cuda"), wt)


def test_against_lpips_package(setup):
    try:
        import lpips
    except ImportError as e:
        pytest.skip(f"the lpips package is not importable ({e})")
    E, _, _ = setup
    net = lpips.LPIPS(net="alex", pretrained=False, pnet_rand=True, verbose=False).eval()
    wt = E.lpips_weights(net)
    gt, gen = R.frames(55, 4, 120, 160)
    with torch.no_grad():
        to = lambda a: 2 * torch.from_numpy(a).permute(0, 3, 1, 2) - 1
        ref = net(to(gt), to(gen)).reshape(-1).double().numpy()   # the package in fp32
    out = E.lpips(*_cuda(gt, gen), wt).cpu().double().numpy()
    assert np.abs(out - ref).max() <= TOL
