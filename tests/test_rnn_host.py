"""CPU tests of the RNN layer on the built-in engine (DESIGN.md section 14): the float64 reference of rnn_ref.py against
a hand-worked case, central finite differences, the float64 PyTorch mirror and every plausible wrong version it lists;
the parser's RNN blobs, fillers, multipliers and shared params; every RNN refusal with Caffe's wording; transposed
CoSData tops; InnerProduct on other axes; and both recurrent fixtures' layouts and plans."""
import math
import os

import numpy as np
import pytest
import torch

import rnn_ref as R
from conftest import ROOT
from test_autoencoder_host import _op_lines
from test_embed_host import _write
from test_native_producer_host import _check_layout

CONFIGS = os.path.join(ROOT, "tests", "golden", "configs")
LM_SOLVER = os.path.join(CONFIGS, "rnn_lm_solver.prototxt")
CAPTION_SOLVER = os.path.join(CONFIGS, "rnn_caption_solver.prototxt")


# --------------------------------------------------------------------------- the reference
def _hand_case():
    """T = 2, N = 1, I = H = 1: cont starts a new sequence at t = 0 and continues at t = 1."""
    W = {"w_xh": np.array([[0.5]]), "b_h": np.array([0.1]), "w_hh": np.array([[2.0]]), "w_ho": np.array([[1.5]]),
         "b_o": np.array([-0.2])}
    x, cont, h0 = np.array([[[1.0]], [[-1.0]]]), np.array([[0.0], [1.0]]), np.array([[0.3]])
    return W, x, cont, h0


def _hand_check(mutation=None):
    W, x, cont, h0 = _hand_case()
    o, h = R.forward(W, x, cont, h0, mutation=mutation)
    h0_, h1 = math.tanh(0.6), math.tanh(2 * math.tanh(0.6) - 0.4)  # h_{-1} = 0.3 is flushed at t = 0
    want_o = [math.tanh(1.5 * h0_ - 0.2), math.tanh(1.5 * h1 - 0.2)]
    if not np.allclose(h[1:].ravel(), [h0_, h1], rtol=1e-14) or not np.allclose(o.ravel(), want_o, rtol=1e-14):
        return False
    g, dx, _, _ = R.backward(W, x, cont, h0, np.ones((2, 1, 1)), mutation=mutation)
    dzo = [1 - v * v for v in want_o]
    dpre1 = dzo[1] * 1.5 * (1 - h1 * h1)
    dpre0 = (dzo[0] * 1.5 + 1.0 * 2.0 * dpre1) * (1 - h0_ * h0_)  # cont_1 = 1 carries dpre_1 W_hh back to h_0
    want = {"w_ho": dzo[0] * h0_ + dzo[1] * h1, "b_o": sum(dzo), "w_hh": dpre0 * 0.0 * 0.3 + dpre1 * 1.0 * h0_,
            "w_xh": dpre0 * 1.0 + dpre1 * -1.0, "b_h": dpre0 + dpre1}
    return (all(np.allclose(g[k].ravel(), [v], rtol=1e-13) for k, v in want.items()) and
            np.allclose(dx.ravel(), [dpre0 * 0.5, dpre1 * 0.5], rtol=1e-13))


def _random_case(rng, T=3, N=2, I=3, H=4, S=2):
    W = {k: rng.randn(*s) * 0.6 for k, s in R.blob_shapes(I, H, S)}
    x, xs = rng.randn(T, N, I), rng.randn(N, S)
    cont = np.array([[0.5, 1.0], [2.0, 0.0], [1.0, 1.0]])[:T]
    return W, x, cont, rng.randn(N, H) * 0.5, xs, rng.randn(T, N, H)


def _fd_check(mutation=None, eps=1e-6):
    """Every gradient of the reference against central differences of its own loss sum(R * o)."""
    rng = np.random.RandomState(5)
    W, x, cont, h0, xs, Rw = _random_case(rng)
    g, dx, dxs, _ = R.backward(W, x, cont, h0, Rw, xs, mutation)

    def loss():
        return float((R.forward(W, x, cont, h0, xs, mutation)[0] * Rw).sum())
    for name, arr, grad in [(k, W[k], g[k]) for k in W] + [("x", x, dx), ("x_static", xs, dxs)]:
        for i in range(arr.size):
            v = arr.flat[i]
            arr.flat[i] = v + eps
            up = loss()
            arr.flat[i] = v - eps
            down = loss()
            arr.flat[i] = v
            if abs((up - down) / (2 * eps) - grad.flat[i]) > 1e-6 * max(1.0, abs(grad.flat[i])):
                return False
    return True


def _torch_calls(flat, I, H, S, calls):
    """The PyTorch mirror in float64 over consecutive calls, the state detached between them."""
    from caffeonspark_b200 import nets
    m = nets.rnn_module(I, H, S).double()
    off = 0
    for p in m.parameters():
        p.data.copy_(torch.from_numpy(flat[off:off + p.numel()]).view_as(p))
        off += p.numel()
    h = torch.zeros(calls[0][1].shape[1], H, dtype=torch.float64)
    out = []
    for x, cont, dtop, xs in calls:
        m.zero_grad()
        xt = torch.from_numpy(x).requires_grad_()
        st = torch.from_numpy(xs).requires_grad_() if xs is not None else None
        o, h = m(xt, torch.from_numpy(cont), h.detach(), st)
        (o * torch.from_numpy(dtop)).sum().backward()
        grads = [p.grad.numpy().copy() for p in m.parameters()]
        out.append((o.detach().numpy(), grads, xt.grad.numpy(), st.grad.numpy() if st is not None else None))
    return out


def _mirror_check(mutation=None):
    """Two consecutive calls of the reference, its blobs unpacked from one flat vector, against the PyTorch mirror."""
    rng = np.random.RandomState(8)
    T, N, I, H, S = 4, 3, 2, 5, 3
    flat = rng.randn(sum(int(np.prod(s)) for _, s in R.blob_shapes(I, H, S))) * 0.5
    W = R.unpack(flat, I, H, S, mutation)
    calls = []
    for c in range(2):
        cont = (rng.rand(T, N) < 0.7).astype(np.float64)
        cont[0, 0] = 1.0  # a stream that continues across the call boundary
        calls.append((rng.randn(T, N, I), cont, rng.randn(T, N, H), rng.randn(N, S)))
    got, _ = R.run_calls(W, calls, mutation=mutation)
    want = _torch_calls(flat, I, H, S, calls)
    for (o, g, dx, dxs), (to, tg, tdx, tdxs) in zip(got, want):
        names = [k for k, _ in R.blob_shapes(I, H, S)]
        if not (np.allclose(o, to, atol=1e-12) and np.allclose(dx, tdx, atol=1e-12) and
                np.allclose(dxs, tdxs, atol=1e-12) and
                all(np.allclose(g[k], tg[j], atol=1e-12) for j, k in enumerate(names))):
            return False
    return True


def _checks(mutation=None):
    return {"hand": _hand_check(mutation), "fd": _fd_check(mutation), "mirror": _mirror_check(mutation)}


def test_the_reference_passes_every_check():
    assert _checks() == {"hand": True, "fd": True, "mirror": True}


@pytest.mark.parametrize("mutation", R.MUTATIONS)
def test_each_mutation_fails_a_check(mutation):
    assert not all(_checks(mutation).values()), mutation


def test_cont_zero_at_the_start_makes_a_call_independent_of_the_last():
    rng = np.random.RandomState(2)
    W, x, cont, _, xs, dtop = _random_case(rng)
    cont[0] = 0
    a = R.run_calls(W, [(x, cont, dtop, xs)])[0][0]
    b = R.run_calls(W, [(x + 1, np.ones_like(cont), dtop, xs), (x, cont, dtop, xs)])[0][1]
    assert np.allclose(a[0], b[0], atol=1e-15) and all(np.allclose(a[1][k], b[1][k], atol=1e-15) for k in W)


# --------------------------------------------------------------------------- the parser and the plan
def _rnn(name, bottoms, top, H, extra="", param=""):
    b = " ".join(f'bottom: "{x}"' for x in bottoms)
    return (f'layer {{ name: "{name}" type: "RNN" {b} top: "{top}" {param} recurrent_param {{ num_output: {H} '
            f'{extra} }} }}\n')


EUCLID = 'layer { name: "loss" type: "EuclideanLoss" bottom: "%s" bottom: "t" top: "l" }'
FILLERS = 'weight_filler { type: "uniform" min: -0.1 max: 0.1 } bias_filler { type: "constant" value: 0.5 }'


@pytest.mark.parametrize("static", [False, True])
def test_rnn_blobs_fillers_and_multipliers(cos, tmp_path, static):
    T, N, I, H, S = 5, 3, 4, 6, 7
    inputs = {"x": (T, N, 2, 2), "cont": (T, N), "t": (T, N, H)}
    if static:
        inputs["xs"] = (N, S)
    param = " ".join(f"param {{ lr_mult: {k + 1} decay_mult: {k} }}" for k in range(6 if static else 5))
    bottoms = ["x", "cont"] + (["xs"] if static else [])
    solver = _write(tmp_path, inputs, _rnn("r", bottoms, "y", H, FILLERS, param) + EUCLID % "y")
    d = cos.parse_solver(solver)
    shapes = [(H, I), (H,)] + ([(H, S)] if static else []) + [(H, H), (H, H), (H,)]
    assert list(d.counts) == [int(np.prod(s)) for s in shapes]
    assert list(d.lr_mult) == [float(k + 1) for k in range(len(shapes))]
    assert list(d.decay_mult) == [float(k) for k in range(len(shapes))]
    text = cos.native_producer_plan(solver)
    blobs = [line.split()[3:] for line in text.splitlines() if line.startswith("blob ")]
    kinds = ["uniform", "constant"] + (["uniform"] if static else []) + ["uniform", "uniform", "constant"]
    assert blobs == [["x".join(map(str, s)), k] for s, k in zip(shapes, kinds)]
    offs = np.cumsum([0] + [int(np.prod(s)) for s in shapes])
    roles = ["w_xh", "b_h"] + (["w_xh_static"] if static else []) + ["w_hh", "w_ho", "b_o"]
    line = _op_lines(text)[0]
    want = (f"op 0 RNN r {T}x{N}x2x2 -> {T}x{N}x{H} T={T} N={N} H={H} cont=1" + (" static=3" if static else "") +
            "".join(f" {r}={o}" for r, o in zip(roles, offs)) + " staged-bottom")
    assert line == want
    _check_layout(cos, text, solver, int(offs[-1]))


def test_two_rnns_share_named_params_and_one_cont(cos, tmp_path):
    param = 'param { name: "wxh" } param { name: "bh" } param { name: "whh" } param { name: "who" } param { name: "bo" }'
    body = (_rnn("r1", ["x", "cont"], "y1", 4, param=param) +
            'layer { name: "sc" type: "Scale" bottom: "y1" top: "s" scale_param { axis: 0 } }\n' +
            _rnn("r2", ["s", "cont"], "y", 4, param=param) + EUCLID % "y")
    solver = _write(tmp_path, {"x": (3, 2, 4), "cont": (3, 2), "t": (3, 2, 4)}, body)
    d = cos.parse_solver(solver)
    assert list(d.counts) == [16, 4, 16, 16, 4, 3]  # the Scale between them has 3
    lines = _op_lines(cos.native_producer_plan(solver))
    assert lines[0] == "op 0 RNN r1 3x2x4 -> 3x2x4 T=3 N=2 H=4 cont=1 w_xh=0 b_h=16 w_hh=20 w_ho=36 b_o=52 staged-bottom"
    assert lines[2] == "op 2 RNN r2 3x2x4 -> 3x2x4 T=3 N=2 H=4 cont=1 w_xh=0 b_h=16 w_hh=20 w_ho=36 b_o=52 shares=0,1,2,3,4"


@pytest.mark.parametrize("body,inputs,match", [
    (_rnn("r", ["x", "cont"], "y", 0), None, r"^layer 'r' \(RNN\): num_output must be positive$"),
    (_rnn("r", ["x1", "cont"], "y", 4), {"x1": (5,)},
     r"^layer 'r' \(RNN\): bottom\[0\] must have at least 2 axes -- \(#timesteps, #streams, \.\.\.\)$"),
    (_rnn("r", ["x", "c3"], "y", 4), {"c3": (5, 3, 1)},
     r"^layer 'r' \(RNN\): bottom\[1\] must have exactly 2 axes -- \(#timesteps, #streams\)$"),
    (_rnn("r", ["x", "c3"], "y", 4), {"c3": (4, 3)},
     r"^layer 'r' \(RNN\): Check failed: T_ == bottom\[1\]->shape\(0\) \(5 vs\. 4\)$"),
    (_rnn("r", ["x", "c3"], "y", 4), {"c3": (5, 2)},
     r"^layer 'r' \(RNN\): Check failed: N_ == bottom\[1\]->shape\(1\) \(3 vs\. 2\)$"),
    (_rnn("r", ["x", "cont", "xs"], "y", 4), {"xs": (2, 7)},
     r"^layer 'r' \(RNN\): Check failed: N_ == bottom\[2\]->shape\(0\) \(3 vs\. 2\)$"),
    (_rnn("r", ["x"], "y", 4), None, r"^layer 'r' \(RNN\): RNN Layer takes at least 2 bottom blob\(s\) as input\.$"),
    (_rnn("r", ["x", "cont", "xs", "t"], "y", 4), {"xs": (3, 7)},
     r"^layer 'r' \(RNN\): RNN Layer takes at most 3 bottom blob\(s\) as input\.$"),
    ('layer { name: "r" type: "RNN" bottom: "x" bottom: "cont" top: "y" top: "y2" recurrent_param { num_output: 4 } }\n',
     None, r"^layer 'r' \(RNN\): RNN Layer produces 1 top blob\(s\) as output\.$"),
])
def test_rnn_parser_refusals(cos, tmp_path, body, inputs, match):
    shapes = {"x": (5, 3, 2), "cont": (5, 3), "t": (5, 3, 4)}
    shapes.update(inputs or {})
    with pytest.raises(cos.CosError, match=match):
        cos.parse_solver(_write(tmp_path, shapes, body + EUCLID % "y"))


def test_rnn_engine_refusals(cos, tmp_path):
    shapes = {"x": (5, 3, 2), "cont": (5, 3), "t": (5, 3, 4), "h0": (1, 3, 4)}
    exposed = ('layer { name: "r" type: "RNN" bottom: "x" bottom: "cont" bottom: "h0" top: "y" top: "hT" '
               'recurrent_param { num_output: 4 expose_hidden: true } }\n')
    for d in "abc":
        (tmp_path / d).mkdir()
    solver = _write(tmp_path / "a", shapes, exposed + EUCLID % "y")
    assert list(cos.parse_solver(solver).counts) == [8, 4, 16, 16, 4]  # the parser lays it out
    with pytest.raises(cos.CosError, match=r"^layer 'r' \(RNN\): expose_hidden: true is not supported \(native "
                                           r"producer\)$"):
        cos.native_producer_plan(solver)
    learned_cont = ('layer { name: "sc" type: "Scale" bottom: "cont" top: "c2" scale_param { axis: 0 } }\n' +
                    _rnn("r", ["x", "c2"], "y", 4))
    with pytest.raises(cos.CosError, match=r"^layer 'r' \(RNN\): Cannot backpropagate to sequence indicators\. "
                                           r"\(native producer\)$"):
        cos.native_producer_plan(_write(tmp_path / "b", shapes, learned_cont + EUCLID % "y"))
    # the same learned cont off the loss is fine: that RNN runs no backward
    off = (learned_cont + _rnn("r2", ["x2", "cont"], "y2", 4) + EUCLID % "y2" +
           '\nlayer { name: "s" type: "Silence" bottom: "y" }')
    lines = _op_lines(cos.native_producer_plan(_write(tmp_path / "c", dict(shapes, x2=(5, 3, 2)), off)))
    assert lines[1].endswith("no-backward") and lines[0].endswith("no-backward")


def _cos_net(tmp_path, tops, batch=8, body=""):
    t = "".join(f'top: "{n}" ' for n, _ in tops)
    spec = "".join(f"top {{ name: \"{n}\" type: INT_ARRAY channels: 6 {extra} }} " for n, extra in tops)
    (tmp_path / "net.prototxt").write_text(
        f'name: "t" layer {{ name: "data" type: "CoSData" {t} cos_data_param {{ batch_size: {batch} {spec} }} }}\n' + body)
    (tmp_path / "solver.prototxt").write_text('net: "net.prototxt"\nbase_lr: 0.01\nlr_policy: "fixed"\n')
    return str(tmp_path / "solver.prototxt")


def test_transposed_cos_data_tops(cos, tmp_path):
    body = ('layer { name: "e" type: "Embed" bottom: "a" top: "ea" embed_param { input_dim: 9 num_output: 2 } }\n'
            'layer { name: "e2" type: "Embed" bottom: "b" top: "eb" embed_param { input_dim: 9 num_output: 2 } }\n'
            'layer { name: "loss" type: "EuclideanLoss" bottom: "ea" bottom: "eb" top: "l" }')
    tops = [("a", "sample_num_axes: 1 transpose: true"), ("b", "sample_num_axes: 1 transpose: true height: 2")]
    solver = _cos_net(tmp_path, tops, 8, body)
    d = cos.parse_solver(solver)
    assert d.batch_size == 8  # not the first top's leading axis, 6
    text = cos.native_producer_plan(solver)
    assert text.startswith("input 0 a 48\ninput 1 b 48\n")
    assert _op_lines(text)[0].startswith("op 0 Embed e 6x8 -> 6x8x2 ")
    (tmp_path / "bad").mkdir()
    with pytest.raises(cos.CosError, match=r"^layer 'data' \(CoSData\): each sample must be a 1d-vector if transpose "
                                           r"is used$"):
        cos.parse_solver(_cos_net(tmp_path / "bad", [("a", "sample_num_axes: 2 height: 3 transpose: true")]))
    (tmp_path / "plain").mkdir()  # transpose: false keeps [batch, ...]
    assert cos.parse_solver(_cos_net(tmp_path / "plain", [("a", "sample_num_axes: 1 transpose: false")])).batch_size == 8


@pytest.mark.parametrize("axis,rows,k", [(0, 1, 120), (2, 6, 20), (3, 24, 5), (-1, 24, 5), (1, 2, 60)])
def test_inner_product_on_any_axis(cos, tmp_path, axis, rows, k):
    body = (f'layer {{ name: "ip" type: "InnerProduct" bottom: "x" top: "y" inner_product_param {{ num_output: 7 '
            f'axis: {axis} }} }}\n')
    shape = (2, 3, 4, 5)
    a = axis % 4
    out = shape[:a] + (7,)
    solver = _write(tmp_path, {"x": shape, "t": out}, body + EUCLID % "y")
    line = _op_lines(cos.native_producer_plan(solver))[0]
    out_text = "x".join(map(str, out))
    assert line == f"op 0 InnerProduct ip 2x3x4x5 -> {out_text} w=0:{7 * k} b={7 * k}:7 staged-bottom"
    assert rows * k == 120


def test_inner_product_transpose_stays_refused(cos, tmp_path):
    body = ('layer { name: "ip" type: "InnerProduct" bottom: "x" top: "y" inner_product_param { num_output: 7 '
            'axis: 2 transpose: true } }\n')
    with pytest.raises(cos.CosError, match=r"layer 'ip' \(InnerProduct\): transpose: true is not supported"):
        cos.native_producer_plan(_write(tmp_path, {"x": (2, 3, 4), "t": (2, 3, 7)}, body + EUCLID % "y"))


# --------------------------------------------------------------------------- the fixtures
def test_the_fixture_layouts(cos):
    from caffeonspark_b200 import nets
    lm = [2000 * 128, 256 * 128, 256, 256 * 256, 256 * 256, 256, 2000 * 256, 2000]
    rnn1 = [128 * 64, 128, 128 * 256, 128 * 128, 128 * 128, 128]
    rnn2 = [128 * 128, 128, 128 * 128, 128 * 128, 128]
    cap = [20 * 25, 20, 50 * 20 * 25, 50, 256 * 800, 256, 1000 * 64] + rnn1 + rnn2 + [1000 * 128, 1000]
    for solver, counts, total, module, batch in ((LM_SOLVER, lm, 934352, nets.rnn_lm_module(), 32),
                                                 (CAPTION_SOLVER, cap, 547018, nets.rnn_caption_module(), 16)):
        assert sum(counts) == total
        d = cos.parse_solver(solver)
        assert d.param_count == total and list(d.counts) == counts and d.batch_size == batch
        assert [p.numel() for p in module.parameters()] == counts
    assert nets.RNN_LM_PARAM_COUNT == 934352 and nets.RNN_CAPTION_PARAM_COUNT == 547018
    assert len(lm) == 8 and len(cap) == 20


LM_OPS = [
    "op 0 Embed embed 20x32 -> 20x32x128 input_dim=2000 num_output=128 w=0:256000 staged-bottom",
    "op 1 RNN rnn 20x32x128 -> 20x32x256 T=20 N=32 H=256 cont=0 w_xh=256000 b_h=288768 w_hh=289024 w_ho=354560 "
    "b_o=420096",
    "op 2 InnerProduct predict 20x32x256 -> 20x32x2000 w=420352:512000 b=932352:2000",
    "op 3 SoftmaxWithLoss loss 20x32x2000 -> scalar axis=2 label=2 loss_weight=1",
]
CAPTION_OPS = [
    "op 0 Convolution conv1 16x1x28x28 -> 16x20x24x24 k5x5 s1x1 p0x0 w=0:500 b=500:20 staged-bottom",
    "op 1 Pooling(MAX) pool1 16x20x24x24 -> 16x20x12x12 k2x2 s2x2 p0x0",
    "op 2 Convolution conv2 16x20x12x12 -> 16x50x8x8 k5x5 s1x1 p0x0 w=520:25000 b=25520:50",
    "op 3 Pooling(MAX) pool2 16x50x8x8 -> 16x50x4x4 k2x2 s2x2 p0x0",
    "op 4 InnerProduct ip1 16x50x4x4 -> 16x256 w=25570:204800 b=230370:256",
    "op 5 ReLU relu1 16x256 -> 16x256 in-place",
    "op 6 Embed embed 12x16 -> 12x16x64 input_dim=1000 num_output=64 w=230626:64000 staged-bottom",
    "op 7 RNN rnn1 12x16x64 -> 12x16x128 T=12 N=16 H=128 cont=1 static=9 w_xh=294626 b_h=302818 w_xh_static=302946 "
    "w_hh=335714 w_ho=352098 b_o=368482",
    "op 8 RNN rnn2 12x16x128 -> 12x16x128 T=12 N=16 H=128 cont=1 w_xh=368610 b_h=384994 w_hh=385122 w_ho=401506 "
    "b_o=417890",
    "op 9 InnerProduct predict 12x16x128 -> 12x16x1000 w=418018:128000 b=546018:1000",
    "op 10 SoftmaxWithLoss loss 12x16x1000 -> scalar axis=2 label=3 loss_weight=1",
]


@pytest.mark.parametrize("solver,ops,inputs,total", [
    (LM_SOLVER, LM_OPS, "input 0 cont_sentence 640\ninput 1 input_sentence 640\ninput 2 target_sentence 640\n", 934352),
    (CAPTION_SOLVER, CAPTION_OPS, "input 0 data 12544\ninput 1 cont_sentence 192\ninput 2 input_sentence 192\n"
     "input 3 target_sentence 192\n", 547018)])
def test_the_fixture_plans(cos, solver, ops, inputs, total):
    text = cos.native_producer_plan(solver)
    assert text.startswith(inputs + "op 0 ")
    assert _op_lines(text) == ops
    _check_layout(cos, text, solver, total)
