"""Host checks of the graph and loss op references in producer_ops_ref.py (Slice, Concat, Split, Eltwise, Scale,
EuclideanLoss, ContrastiveLoss) that test_gpu_producer_graph_ops.py holds the built-in producer to: they agree with
torch float64 where Caffe and PyTorch agree, follow Caffe on hand-worked cases where they do not, and each bound admits
an fp32 evaluation in the engine's order while rejecting a subtly wrong one.  Also the plan's side of the GPU cases:
Scale's outer / dim / inner and the Slice and Concat ranges (DESIGN.md section 14)."""
import numpy as np
import pytest
import torch

import producer_ops_ref as R
import test_gpu_producer_graph_ops as G
from caffeonspark_b200 import nets
from test_gpu_producer_ops import _net

F32 = np.float32


def _t(a):
    return torch.tensor(np.asarray(a, np.float64), requires_grad=True)


# --------------------------------------------------------------------------- references against torch float64
def test_slice_and_concat_match_torch():
    rng = np.random.RandomState(1)
    x = R.gaussian(rng, (3, 7, 4, 9))
    for axis, ranges in ((1, R.slice_bounds(7, [2, 3, 6])), (3, R.slice_bounds(9, tops=3)), (0, R.slice_bounds(3, [1]))):
        parts = R.slice_forward(x, axis, ranges)
        ref = torch.split(torch.from_numpy(x), [e - b for b, e in ranges], dim=axis)
        assert all(np.array_equal(p, t.numpy()) for p, t in zip(parts, ref))
        assert np.array_equal(np.concatenate(parts[::-1], axis), torch.cat(ref[::-1], axis).numpy())


@pytest.mark.parametrize("shape,axis,num_axes", [((4, 3, 5, 6), 1, 1), ((4, 3, 5, 6), 2, 2), ((4, 3, 5, 6), 1, 0),
                                                 ((7, 33), 0, -1), ((4, 3, 5, 6), 3, 1)])
def test_scale_matches_a_broadcast_multiply(shape, axis, num_axes):
    rng = np.random.RandomState(len(shape) + axis)
    view = R.scale_view(shape, axis, num_axes)
    end = len(shape) if num_axes == -1 else axis + num_axes
    x, s, b = R.gaussian(rng, shape), R.gaussian(rng, shape[axis:end]), R.gaussian(rng, shape[axis:end])
    bshape = (1,) * axis + shape[axis:end] + (1,) * (len(shape) - end)
    xt, st, bt = _t(x), _t(s), _t(b)
    yt = xt * st.reshape(bshape) + bt.reshape(bshape)
    y, _ = R.scale_forward(x, s, b, view)
    np.testing.assert_allclose(y, yt.detach().numpy(), rtol=1e-15)
    dy = R.gaussian(rng, shape)
    yt.backward(torch.from_numpy(dy.astype(np.float64)))
    ds, _, db, _, dx = R.scale_backward(x, s, dy, view)
    np.testing.assert_allclose(ds, st.grad.numpy().ravel(), rtol=1e-12)
    np.testing.assert_allclose(db, bt.grad.numpy().ravel(), rtol=1e-12)
    np.testing.assert_allclose(dx, xt.grad.numpy(), rtol=2 * R.U)


def test_eltwise_matches_torch_autograd():
    rng = np.random.RandomState(2)
    xs = [R.gaussian(rng, (5, 7)) for _ in range(3)]
    dy = R.gaussian(rng, (5, 7)).astype(np.float64)
    ts = [_t(x) for x in xs]
    (0.5 * ts[0] - 1.5 * ts[1] + ts[2]).backward(torch.from_numpy(dy))
    y, _ = R.eltwise_sum(xs, (0.5, -1.5, 1))
    x64 = [x.astype(np.float64) for x in xs]
    np.testing.assert_allclose(y, 0.5 * x64[0] - 1.5 * x64[1] + x64[2], rtol=1e-15)
    for t, c in zip(ts, (0.5, -1.5, 1)):
        np.testing.assert_allclose(R.eltwise_sum_backward32(dy, c), t.grad.numpy(), rtol=R.U)
    ts = [_t(x) for x in xs]
    (ts[0] * ts[1] * ts[2]).backward(torch.from_numpy(dy))
    for stable in (True, False):
        for (g, _), t in zip(R.eltwise_prod_backward(xs, dy, stable), ts):
            np.testing.assert_allclose(g, t.grad.numpy(), rtol=1e-15)
    ts = [_t(x) for x in xs]
    torch.stack(ts).amax(0).backward(torch.from_numpy(dy))  # no ties in Gaussian draws
    y, win = R.eltwise_max(xs)
    assert np.array_equal(y, np.max(xs, axis=0))
    for g, t in zip(R.eltwise_max_backward(dy, win, 3), ts):
        np.testing.assert_array_equal(g, t.grad.numpy().astype(F32))


@pytest.mark.parametrize("lw", [1.0, 0.5, 3.0])
def test_euclidean_matches_mse(lw):
    rng = np.random.RandomState(3)
    a, b = R.gaussian(rng, (7, 3, 4)), R.gaussian(rng, (7, 12))
    at, bt = _t(a), _t(b.reshape(a.shape))
    lt = lw * ((at - bt) ** 2).sum() / 7 / 2
    lt.backward()
    loss, _ = R.euclidean_loss(a, b, lw)
    assert loss == pytest.approx(lt.item(), rel=1e-14)
    da, db = R.euclidean_grads32(a, b, lw)
    np.testing.assert_allclose(da, at.grad.numpy(), rtol=3 * R.U)
    np.testing.assert_allclose(db, bt.grad.numpy().reshape(b.shape), rtol=3 * R.U)


@pytest.mark.parametrize("legacy", [False, True])
def test_contrastive_matches_nets(legacy):
    rng = np.random.RandomState(4 + legacy)
    a, b = R.gaussian(rng, (40, 3), 0.4), R.gaussian(rng, (40, 3), 0.4)
    sim = G.SIMS[np.arange(40) % 8]
    at, bt = _t(a), _t(b)
    lt = nets.contrastive_loss(at, bt, torch.from_numpy(sim.astype(np.float64)), 1.0, legacy, 2.0)
    lt.backward()
    loss, da, db, _ = R.contrastive_loss(a, b, sim, 1.0, legacy, 2.0, eps=1e-4)  # nets adds a float64 1e-4
    assert loss == pytest.approx(lt.item(), rel=1e-14)
    np.testing.assert_allclose(da, at.grad.numpy(), rtol=1e-12, atol=1e-300)
    np.testing.assert_allclose(db, bt.grad.numpy(), rtol=1e-12, atol=1e-300)


# --------------------------------------------------------------------------- Caffe's rules, hand-worked
def test_eltwise_max_tie_and_nan_rule():
    nan, inf = np.nan, np.inf
    x0 = np.array([1, 2, nan, 1, 1, -inf, 3], F32)
    x1 = np.array([1, 1, 5, nan, 1, -inf, 3], F32)
    x2 = np.array([1, 2, 6, 7, 2, -inf, nan], F32)
    y, win = R.eltwise_max([x0, x1, x2])
    # a tie of 0 and 1 goes to 1; a later tie stays; NaN in bottom 0 loses to bottom 1, NaN as bottom 1 wins and
    # nothing is > NaN; a later NaN never takes over
    assert win.tolist() == [1, 0, 2, 1, 2, 1, 1]
    assert np.array_equal(y, np.array([1, 2, 6, nan, 2, -inf, 3], F32), equal_nan=True)
    _, last = R.eltwise_max([x0, x1, x2], later_wins_ties=True)
    assert last.tolist() == [2, 2, 2, 1, 2, 2, 1]


def test_contrastive_truncates_sim_and_zeroes_at_the_margin():
    a = np.array([[1.0, 0.0]] * 8, F32)
    b = np.zeros((8, 2), F32)
    loss, da, _, mdist = R.contrastive_loss(a, b, G.SIMS, margin=1.0, legacy=True)
    # sims 0 0.5 0.999 -0.5 truncate to 0 (dissimilar, mdist = 0: no loss, no gradient); 1 1.5 2 -1 are similar
    assert np.all(mdist == 0)
    assert (da[:, 0] != 0).tolist() == [False, True, False, False, True, False, True, True]
    assert loss == 4 * 1.0 / 8 / 2
    _, da, _, _ = R.contrastive_loss(a, b, G.SIMS, margin=2.0, legacy=True)
    assert da[0].tolist() == [-1 / 8, 0]  # mdist 1 > 0: -alpha * d
    _, da, _, _ = R.contrastive_loss(a, b, G.SIMS, margin=2.0, legacy=False)
    assert da[0, 0] == pytest.approx(-1 / 8 * 1.0 / (1 + R.EPS_DIST), rel=1e-15)


def test_contrastive_non_finite_rule():
    a = np.array([[np.nan, 0.0], [np.inf, 0.0], [np.nan, 1.0]], F32)
    b = np.zeros((3, 2), F32)
    for legacy in (False, True):
        loss, da, db, _ = R.contrastive_loss(a[:2], b[:2], np.zeros(2, F32), legacy=legacy)
        assert np.isnan(loss) and not da.any() and not db.any()  # NaN reaches the loss; exact-0 gradients
        loss, da, _, _ = R.contrastive_loss(a[1:2], b[1:2], np.zeros(1, F32), legacy=legacy)
        assert loss == 0 and not da.any()  # inf: mdist = -inf adds 0
        loss, da, _, _ = R.contrastive_loss(a[2:], b[2:], np.ones(1, F32), legacy=legacy)
        assert np.isnan(loss) and np.isnan(da[0, 0]) and da[0, 1] == 1.0  # similar: alpha * d


def test_prod_y_over_x_nans():
    x0 = np.array([0, 2, np.inf, 3, 0], F32)
    x1 = np.array([5, 0, 2, 4, np.inf], F32)
    dy = np.ones(5)
    (g0, _), (g1, _) = R.eltwise_prod_backward([x0, x1], dy, stable=False)
    # caffe_div(y, x): 0/0, inf/inf and (0 * inf)/x are NaN; 0 / 2 and inf / 2 are not
    assert np.isnan(g0).tolist() == [True, False, True, False, True]
    assert np.isnan(g1).tolist() == [False, True, False, False, True]
    assert g0[1] == 0 and g1[2] == np.inf and g0[3] == 4
    (s0, _), _ = R.eltwise_prod_backward([x0, x1], dy, stable=True)
    assert s0[0] == 5 and s0[1] == 0


def test_split_sums_in_top_order():
    ds = [np.array([1.0], F32), np.array([2.0 ** -24], F32), np.array([2.0 ** -24], F32)]
    assert R.split_backward32(ds)[0] == 1.0  # (1 + u) rounds to even, twice
    assert R.split_backward32(ds, reverse=True)[0] == 1.0 + 2.0 ** -23  # u + u first


# --------------------------------------------------------------------------- the bounds: admit fp32, reject mutations
def _outside(got, ref, bound):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return np.abs(got - ref) > bound


def _admits(got32, ref, bound, what):
    assert not _outside(got32, ref, bound).any(), f"{what}: the bound rejects an fp32 evaluation"


def _rejects(mutated, ref, bound, what, right=None):
    """Most elements the mutation changes (from `right`, the correct evaluation, or else the reference) fall outside
    the bound."""
    m = np.asarray(mutated, np.float64)
    changed = m != (ref if right is None else np.asarray(right, np.float64))
    assert changed.any(), f"{what}: the mutation changes nothing"
    frac = _outside(m, ref, bound)[changed].mean()
    assert frac > 0.5, f"{what}: only {frac:.2f} of the changed elements fall outside the bound"


def test_split_bound_admits_top_order_and_the_fp32_check_rejects_reverse():
    rng = np.random.RandomState(7)
    ds = [R.gaussian(rng, (4000,)) * np.exp2(rng.randint(-12, 12, 4000)).astype(F32) for _ in range(3)]
    ref = sum(d.astype(np.float64) for d in ds)
    _admits(R.split_backward32(ds), ref, R.split_backward_bound(ds), "split")
    _admits(R.split_backward32(ds, reverse=True), ref, R.split_backward_bound(ds), "split reversed")
    # the order is caught by the fp32 equality the GPU test adds, on inputs where the two orders differ
    assert np.mean(R.split_backward32(ds) != R.split_backward32(ds, reverse=True)) > 0.05


def test_scale_bound_admits_one_rounding_and_rejects_two():
    rng = np.random.RandomState(8)
    shape, view = (8, 16, 32), R.scale_view((8, 16, 32), 1, 1)
    x, s, b = R.gaussian(rng, shape), R.gaussian(rng, (16,)), R.gaussian(rng, (16,))
    y, by = R.scale_forward(x, s, b, view)
    # one rounding of the exact x * s + b (float64 holds it exactly when the exponents are close, as here mostly)
    one = (x.astype(np.float64) * s[None, :, None] + b[None, :, None]).astype(F32)
    _admits(one, y, by, "fma")
    two, _ = R.scale_forward(x, s, b, view, two_roundings=True)
    _rejects(two.astype(F32), y, by, "x * s rounded, then + b", right=one)
    ds, bs, db, bb, _ = R.scale_backward(x, s, y, view)
    dy32 = y.astype(F32)
    ds32 = np.zeros(16, F32)
    for i in range(8):  # one fp32 accumulation in a different order still fits
        ds32 += (dy32[i] * x[i]).astype(F32).sum(axis=1, dtype=F32)
    _admits(ds32, ds, bs, "ds")


def test_eltwise_bounds_admit_fp32_and_reject_later_ties():
    rng = np.random.RandomState(9)
    xs = [R.gaussian(rng, (3000,)) for _ in range(4)]
    coeffs = (1, 0.1, -1.5, 0)
    y, by = R.eltwise_sum(xs, coeffs)
    acc = F32(coeffs[0]) * xs[0]
    for c, x in zip(coeffs[1:], xs[1:]):
        acc = (np.float64(F32(c)) * x + acc.astype(np.float64)).astype(F32)  # the fma, rounded once
    _admits(acc, y, by, "SUM")
    p, bp = R.eltwise_prod(xs)
    _admits(xs[0] * xs[1] * xs[2] * xs[3], p, bp, "PROD")
    xd = [R.dyadic(rng, (3000,), top=1) for _ in range(4)]
    dy = R.gaussian(rng, (3000,))
    y, win = R.eltwise_max(xd)
    _, late = R.eltwise_max(xd, later_wins_ties=True)
    assert np.any(win != late)
    right, wrong = R.eltwise_max_backward(dy, win, 4), R.eltwise_max_backward(dy, late, 4)
    _rejects(np.concatenate(wrong), np.concatenate(right).astype(np.float64), 0.0, "later bottom wins ties")


def test_euclidean_bound_admits_fp32_and_rejects_loss_weight_for_alpha():
    rng = np.random.RandomState(10)
    a, b = R.gaussian(rng, (7, 1200)), R.gaussian(rng, (7, 1200))
    loss, bound = R.euclidean_loss(a, b, 3.0)
    d = np.concatenate([(a - b).ravel(), np.zeros(-a.size % 256, F32)])
    part = np.zeros(256, F32)
    for i in range(0, d.size, 256):  # per-thread sums in index order
        part += d[i:i + 256] * d[i:i + 256]
    while part.size > 1:  # the fixed tree
        part = part[:part.size // 2] + part[part.size // 2:]
    got = F32(3.0) * ((part[0] / F32(7)) / F32(2))
    assert abs(float(got) - loss) <= bound
    assert abs(float(F32(3.0) * ((part[0] / F32(1)) / F32(2))) - loss) > bound  # the mutation: / 1
    da, _ = R.euclidean_grads32(a, b, 3.0)
    assert np.all(da != R.euclidean_grads32(a, b, 3.0 * 7)[0] / 1)


@pytest.mark.parametrize("legacy", [False, True])
def test_contrastive_bounds_admit_fp32_and_reject_mutations(legacy):
    rng = np.random.RandomState(11 + legacy)
    n, c, margin = 600, 5, 1.0
    sd = np.sqrt(margin / (2 * c)) if legacy else margin / np.sqrt(2 * c)
    a, b = R.gaussian(rng, (n, c), sd), R.gaussian(rng, (n, c), sd)
    sim = G.SIMS[np.arange(n) % 8]
    loss, da, _, mdist = R.contrastive_loss(a, b, sim, margin, legacy, 2.0)
    lb, gb, e_md = R.contrastive_bounds(a, b, sim, margin, legacy, 2.0)
    dis = np.trunc(sim) == 0
    assert np.all(np.abs(mdist[dis]) > e_md[dis])
    # fp32 in the kernel's order
    d = (a - b).astype(F32)
    dsq = np.zeros(n, F32)
    for j in range(c):
        dsq = dsq + d[:, j] * d[:, j]
    alpha = F32(2.0) / F32(n)
    if legacy:
        md = F32(margin) - dsq
        per = np.where(dis, np.maximum(md, 0), dsq)
        scale = np.where(dis, np.where(md > 0, -alpha, 0), alpha).astype(F32)
    else:
        dist = np.sqrt(dsq)
        md = F32(margin) - dist
        per = np.where(dis, np.maximum(md, 0) * np.maximum(md, 0), dsq)
        beta = ((-alpha) * md) / (dist + F32(1e-4))
        scale = np.where(dis, np.where(md > 0, beta, 0), alpha).astype(F32)
    g32 = scale[:, None] * d
    _admits(g32, da, gb, "da")
    got = F32(2.0) * ((per.astype(F32).sum(dtype=F32) / F32(n)) / F32(2))
    assert abs(float(got) - loss) <= lb
    if legacy:
        _, wrong, _, _ = R.contrastive_loss(a, b, sim, margin, True, 2.0, legacy_grad_without_d=True)
        _rejects(wrong, da, gb, "legacy gradient without d")
    else:
        _, wrong, _, _ = R.contrastive_loss(a, b, sim, margin, False, 2.0, eps=0.0)
        _rejects(wrong, da, gb, "no + 1e-4")


# --------------------------------------------------------------------------- the plan
def _plan(cos, tmp_path, xs, body, staged=None):
    (tmp_path / "net.prototxt").write_text(_net(xs, body, staged=staged)[0])
    return cos.native_producer_plan(str(tmp_path / "net.prototxt"))


def _lines(text, kind):
    return [ln for ln in text.splitlines() if ln.startswith("op ") and ln.split()[2].startswith(kind)]


@pytest.mark.parametrize("shape,param,axis,num_axes", G.SCALE_CASES)
def test_plan_scale_view(cos, tmp_path, shape, param, axis, num_axes):
    body, _ = G.scale_body(param, True, False)
    body += ('layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "st" }\n')
    text = _plan(cos, tmp_path, [np.zeros(shape, F32)], body, staged={"st": np.zeros(shape, F32)})
    outer, dim, inner = R.scale_view(shape, axis, num_axes)
    line = [ln for ln in _lines(text, "Scale") if " sc " in ln][0]
    assert f" outer={outer} dim={dim} inner={inner}" in line, line


@pytest.mark.parametrize("shape,param,axis,ranges,unread", G.SLICE_CASES)
def test_plan_slice_ranges(cos, tmp_path, shape, param, axis, ranges, unread):
    body, gathered = G.slice_body(param, len(ranges), unread, axis)
    parts = R.slice_forward(np.zeros(shape, F32), axis, ranges)
    y = np.concatenate([parts[int(t[1:])] for t in gathered], axis=axis)
    body += 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "st" }\n'
    text = _plan(cos, tmp_path, [np.zeros(shape, F32)], body, staged={"st": y})
    assert [ln.split("axis=")[1] for ln in _lines(text, "Slice")] == [f"{axis} begin={b}" for b, _ in ranges]
    sizes = [ranges[int(t[1:])][1] - ranges[int(t[1:])][0] for t in gathered]
    assert [ln.split("axis=")[1] for ln in _lines(text, "Concat")] == \
        [f"{axis} begin={sum(sizes[:i])}" for i in range(len(sizes))]


@pytest.mark.parametrize("shapes,param,axis,staged", G.CONCAT_CASES)
def test_plan_concat_ranges(cos, tmp_path, shapes, param, axis, staged):
    injected = [np.zeros(s, F32) for i, s in enumerate(shapes) if i != staged]
    y = np.concatenate([np.zeros(s, F32) for s in shapes], axis=axis)
    body = G.concat_body(len(injected), staged, param)
    body += 'layer { name: "loss" type: "EuclideanLoss" bottom: "y" bottom: "t" }\n'
    st = {"t": y} if staged is None else {"st": np.zeros(shapes[staged], F32), "t": y}
    text = _plan(cos, tmp_path, injected, body, staged=st)
    begins = np.cumsum([0] + [s[axis] for s in shapes])[:-1]
    lines = _lines(text, "Concat")
    assert [ln.split("axis=")[1].split()[:2] for ln in lines] == [[str(axis), f"begin={b}"] for b in begins]
    if staged is not None:
        assert "staged-bottom" in lines[staged] and "staged-bottom" not in lines[staged - 1 if staged else 1]


def test_nets_contrastive_loss_follows_the_non_finite_rule():
    """the torch reference of the siamese tests agrees with the kernel's rule on NaN and infinite embeddings"""
    a = np.array([[np.nan, 0.0], [np.inf, 0.0], [np.nan, 1.0], [0.25, 0.5]], F32)
    b = np.zeros((4, 2), F32)
    sim = np.array([0, 0, 1, 0], F32)
    for legacy in (False, True):
        at, bt = _t(a), _t(b)
        lt = nets.contrastive_loss(at, bt, torch.from_numpy(sim.astype(np.float64)), 1.0, legacy)
        lt.backward()
        loss, da, db, _ = R.contrastive_loss(a, b, sim, 1.0, legacy, eps=1e-4)
        assert np.isnan(lt.item()) and np.isnan(loss)
        np.testing.assert_array_equal(at.grad.numpy(), da)
        np.testing.assert_array_equal(bt.grad.numpy(), db)
        assert not at.grad.numpy()[:2].any()
