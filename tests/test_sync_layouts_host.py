"""The named sync layouts (tests/sync_layouts.py) on the host: their properties, the C oracle against the numpy
restatements on every one of them, numpy mutations of the update that they expose and the old power-of-two layouts
do not, and the rounding of parsed multipliers.  No GPU needed."""
from fractions import Fraction

import numpy as np
import pytest

import sync_layouts as S

F = np.float32
SGD_HP = dict(lr_policy="inv", base_lr=0.01, gamma=0.0001, power=0.75, momentum=0.9, weight_decay=0.0005)
ADAM_HP = dict(lr_policy="fixed", base_lr=0.001, momentum=0.9, weight_decay=0.0005, momentum2=0.999, delta=1e-8)

# the layouts the sync tests used before, all multipliers in {0, 0.25, 0.5, 1, 2}
EXISTING = {
    "lenet": ([500, 20, 25000, 50, 400000, 500, 5000, 10], [1, 2] * 4, [1, 1] * 4),
    "cifar10_quick": ([2400, 32, 25600, 32, 51200, 64, 65536, 64, 640, 10], [1, 2] * 5, [1, 1] * 5),
    "ragged_tiny_blobs": ([3, 1, 2, 5, 1, 1, 7, 1021, 2, 1], [1, 2, 1, 2, 1, 2, 1, 2, 1, 2],
                          [1, 0, 1, 0, 1, 0, 1, 1, 0, 1]),
    "single_element": ([1], [1], [1]),
    "not_multiple_of_4": ([4099], [1], [1]),
    "adam_multi": ([5000, 20, 2500, 50, 7, 1021], [1, 2, 1, 2, 1, 2], [1, 0, 1, 0, 1, 1]),
    "l1_multi": ([1021, 7, 64], [1, 2, 1], [1, 0, 0.5]),
}


@pytest.fixture(scope="module")
def adam(oracle):
    from oracle import adam as A
    A.build()
    A.lib()
    return A


@pytest.fixture(scope="module")
def accum(oracle):
    from oracle import accum as A
    A.build()
    A.lib()
    return A


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, F).view(np.uint32), np.asarray(b, F).view(np.uint32))


# ------------------------------------------------------------------ properties

def test_the_named_layouts_are_what_their_names_say():
    for n in S.SEG_SIZES:
        assert len(S.layout(f"seg_{n}")[0]) == n
    c, lm, dm = S.layout("resnet152_bn_like")
    assert len(c) == S.RESNET152_BLOBS == 932
    assert 10 ** 6 <= sum(c) <= 4 * 10 ** 6
    assert lm[-2:] == [10.0, 20.0] and lm[-7:-4] == [0.0, 0.0, 0.0]   # classifier; the last BatchNorm is frozen
    c, _, _ = S.layout("empty_blobs")
    e = S.ends(c)
    assert c[0] == 0 and c[-1] == 0 and any(c[k] == c[k + 1] == 0 for k in range(len(c) - 1))
    # a zero-count blob between two non-empty blobs whose elements share one float4
    assert any(c[k] == 0 and c[k - 1] > 0 and c[k + 1] > 0 and e[k] % 4 != 0 for k in range(1, len(c) - 1))
    for r in (1, 2, 3):
        assert sum(S.layout(f"adam_odd_p_{r}")[0]) % 4 == r
    for name in S.NAMES:
        c, lm, dm = S.layout(name)
        assert len(c) == len(lm) == len(dm) and min(c) >= 0
        assert set(lm) <= set(S.LR_MULTS) and set(dm) <= set(S.DECAY_MULTS)
        assert S.layout(name) == S.layout(name)                              # deterministic


@pytest.mark.parametrize("name", S.NAMES)
def test_shards_cut_blobs_and_float4s_straddle_blob_ends(oracle, name):
    c, _, _ = S.layout(name)
    P = sum(c)
    for N in (2, 3, 4, 8):
        assert S.shard_cuts_inside_a_blob(c, N, oracle.chunk), (name, N)
        if name in S.SEG_NAMES or name == "empty_blobs":
            # in the vector body of some shard (the kernels' fast path), not only in the scalar edges
            best = max(S.max_ends_in_a_float4(c, *_span(oracle.chunk(P, N, r))) for r in range(N))
            assert best >= 3, (name, N, best)
    assert S.max_ends_in_a_float4(c) >= 2


def _span(offset_size):
    o, s = offset_size
    return o, o + s


def _lrc(rate, lm, corr, swapped=False):
    """Adam's per-blob rate: (rate * lr_mult) * correction as the solver rounds it, or rate * (lr_mult * correction)."""
    lm = np.asarray(lm, F)
    return F(rate) * (lm * F(corr)) if swapped else (F(rate) * lm) * F(corr)


@pytest.mark.parametrize("name", S.NAMES)
def test_first_step_multipliers_round_differently_in_the_other_order(adam, name):
    c, lm, _ = S.layout(name)
    corr = adam.adam_correction(ADAM_HP["momentum"], ADAM_HP["momentum2"], 0)
    a, b = _lrc(ADAM_HP["base_lr"], lm, corr), _lrc(ADAM_HP["base_lr"], lm, corr, swapped=True)
    differ = (a != b) & (np.asarray(c) > 0)
    assert differ.any(), name


def test_power_of_two_multipliers_never_round_differently(adam):
    corr = adam.adam_correction(ADAM_HP["momentum"], ADAM_HP["momentum2"], 0)
    for c, lm, _ in EXISTING.values():
        for rate in (0.001, 0.01, 0.0123):
            assert np.array_equal(_lrc(rate, lm, corr), _lrc(rate, lm, corr, swapped=True))


# ------------------------------------------------- C oracle == numpy restatement

def _sgd_case(oracle, name, N, reg, seed):
    c, lm, dm = S.layout(name)
    return oracle.Simulation(N, c, lm, dm, seed=seed, regularization_type=reg, **SGD_HP)


@pytest.mark.parametrize("name", S.NAMES)
@pytest.mark.parametrize("reg", ["L2", "L1"])
def test_c_oracle_equals_numpy_sgd(oracle, name, reg):
    from oracle import numpy_oracle as NO
    for N in range(1, 9):
        sim = _sgd_case(oracle, name, N, reg, seed=11 + N)
        if reg == "L1":
            sim.data[0][:3] = [0.0, -0.0, 0.5]
        d, h = [x.copy() for x in sim.data], [x.copy() for x in sim.hist]
        for t in range(2):
            grads = [sim.gradient(r, t) for r in range(N)]
            rate = sim.rate()
            d, h = NO.step(d, grads, h, sim.counts, sim.lr_mult, sim.decay_mult, rate, sim.hp["momentum"],
                           sim.hp["weight_decay"], reg)
            sim.step(grads)
            for r in range(N):
                assert _bits_equal(sim.data[r], d[r]), (name, reg, N, t, r)
                assert _bits_equal(sim.hist[r], h[r]), (name, reg, N, t, r)


def _adam_worlds(name):
    return (1, 3) if name == "resnet152_bn_like" else (1, 2, 3, 8)


@pytest.mark.parametrize("name", S.NAMES)
def test_c_oracle_equals_numpy_adam(adam, name):
    from oracle import numpy_adam as NA
    c, lm, dm = S.layout(name)
    for N in _adam_worlds(name):
        reg = "L1" if N == 3 else "L2"
        sim = adam.AdamSimulation(N, c, lm, dm, seed=23 + N, regularization_type=reg, **ADAM_HP)
        d, h = [x.copy() for x in sim.data], [x.copy() for x in sim.hist]
        for t in range(2):
            grads = [sim.gradient(r, t) for r in range(N)]
            d, h = NA.step_adam(d, grads, h, c, lm, dm, sim.rate(), ADAM_HP["momentum"], ADAM_HP["momentum2"],
                                ADAM_HP["delta"], ADAM_HP["weight_decay"], sim.iter, reg)
            sim.step(grads)
            P = sim.P
            for r in range(N):
                o, s = adam.O.chunk(P, N, r)
                assert _bits_equal(sim.data[r][o:o + s], d[r][o:o + s]), (name, N, t, r)
                assert _bits_equal(sim.hist[r][o:o + s], h[r][o:o + s]), (name, N, t, r)
                assert _bits_equal(sim.hist[r][P + o:P + o + s], h[r][P + o:P + o + s]), (name, N, t, r)


@pytest.mark.parametrize("name", S.NAMES)
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_c_oracle_equals_numpy_iter_size_3(accum, name, solver):
    from oracle import numpy_accum as NAc
    c, lm, dm = S.layout(name)
    hp = SGD_HP if solver == "SGD" else ADAM_HP
    for N in ((1, 3) if solver == "Adam" and name == "resnet152_bn_like" else (1, 2, 4)):
        sim = accum.AccumSimulation(N, c, lm, dm, iter_size=3, solver_type=solver, seed=31 + N, **hp)
        d, h = [x.copy() for x in sim.data], [x.copy() for x in sim.hist]
        for t in range(2):
            per_pass = [[sim.pass_gradient(r, t, q) for r in range(N)] for q in range(3)]
            acc = accum.accumulate(per_pass)
            assert all(_bits_equal(a, b) for a, b in zip(acc, NAc.accumulate(per_pass)))
            d, h = NAc.step_accum(d, acc, h, c, lm, dm, sim.rate(), hp["momentum"], hp["weight_decay"], 3, sim.iter,
                                  "L2", solver, hp.get("momentum2", 0.999), hp.get("delta", 1e-8))
            sim.step_accumulated(acc)
            P = sim.P
            for r in range(N):
                o, s = accum.O.chunk(P, N, r)
                assert _bits_equal(sim.data[r][o:o + s], d[r][o:o + s]), (name, solver, N, t, r)
                assert _bits_equal(sim.hist[r][o:o + s], h[r][o:o + s]), (name, solver, N, t, r)
                if solver == "Adam":
                    assert _bits_equal(sim.hist[r][P + o:P + o + s], h[r][P + o:P + o + s]), (name, N, t, r)


# ------------------------------------------------------------------ mutations
# One local (N = 1) step from the oracle's seeded start, restated with per-ELEMENT multipliers so that the kernels'
# ways of going wrong can be written down: (a) Adam's rate as rate * (lr_mult * correction), (b) a float4 that
# straddles blob ends updated with its first element's multipliers, (c) lr_mult and decay_mult swapped.

def _element_mults(counts, lm, dm, first_of_float4=False):
    blob = S.blob_of_element(counts)
    if first_of_float4:  # the kernels' vector body at N = 1 is [0, 4*floor(P/4)); the tail is scalar
        body = len(blob) // 4 * 4
        blob = blob.copy()
        blob[:body] = blob[:body:4].repeat(4)
    return np.asarray(lm, F)[blob], np.asarray(dm, F)[blob]


def _local_step(w, g, h, lm_e, dm_e, rate, hp, solver, lrc_swapped=False):
    """One ApplyUpdate at N = 1 in float32 numpy with per-element multipliers; returns (w, history)."""
    ld = F(hp["weight_decay"]) * dm_e
    g = np.where(ld != 0, ld * w + g, g).astype(F)
    if solver == "SGD":
        h = (F(rate) * lm_e * g + (F(hp["momentum"]) * h).astype(F)).astype(F)
        return (F(-1.0) * h + w).astype(F), h
    from oracle import numpy_adam as NA
    P = w.size
    b1, b2 = F(hp["momentum"]), F(hp["momentum2"])
    corr = NA.adam_correction(b1, b2, 0)
    lrc = (F(rate) * (lm_e * F(corr)).astype(F)) if lrc_swapped else ((F(rate) * lm_e).astype(F) * F(corr))
    m = ((F(1) - b1) * g + (b1 * h[:P]).astype(F)).astype(F)
    v = ((F(1) - b2) * (g * g).astype(F) + (b2 * h[P:]).astype(F)).astype(F)
    t = (m / (NA._powf_half(v) + F(hp["delta"])).astype(F)).astype(F)
    return (F(-1.0) * (lrc.astype(F) * t).astype(F) + w).astype(F), np.concatenate([m, v])


def _oracle_first_step(oracle, adam, counts, lm, dm, solver):
    if solver == "SGD":
        sim = oracle.Simulation(1, counts, lm, dm, seed=5, **SGD_HP)
    else:
        sim = adam.AdamSimulation(1, counts, lm, dm, seed=5, **ADAM_HP)
    w0, h0, g = sim.data[0].copy(), sim.hist[0].copy(), sim.gradient(0, 0)
    rate = sim.rate()
    sim.step([g])
    return (w0, g, h0, rate), (sim.data[0], sim.hist[0])


def _mutants(oracle, adam, counts, lm, dm, solver):
    """{"none" | "a" | "b" | "c": whether that variant's first step differs from the oracle's}"""
    (w0, g, h0, rate), (w_ref, h_ref) = _oracle_first_step(oracle, adam, counts, lm, dm, solver)
    hp = SGD_HP if solver == "SGD" else ADAM_HP
    variants = {"none": (_element_mults(counts, lm, dm), False),
                "b": (_element_mults(counts, lm, dm, first_of_float4=True), False),
                "c": (_element_mults(counts, dm, lm), False)}
    if solver == "Adam":
        variants["a"] = (_element_mults(counts, lm, dm), True)
    out = {}
    for k, ((lm_e, dm_e), swapped) in variants.items():
        w, h = _local_step(w0, g, h0, lm_e, dm_e, rate, hp, solver, lrc_swapped=swapped)
        out[k] = not (_bits_equal(w, w_ref) and _bits_equal(h, h_ref))
    return out


@pytest.mark.parametrize("name", S.NAMES)
@pytest.mark.parametrize("solver", ["SGD", "Adam"])
def test_mutations_are_caught_on_the_named_layouts(oracle, adam, name, solver):
    c, lm, dm = S.layout(name)
    got = _mutants(oracle, adam, c, lm, dm, solver)
    assert got["none"] is False, "the per-element restatement must equal the oracle"
    assert got["b"] and got["c"], (name, solver, got)
    if solver == "Adam":
        assert got["a"], (name, got)


# every blob end a multiple of 4 (or one blob): no float4 straddles two blobs.  The others (LeNet's 50-element ip1
# bias ends at 25570) do see mutation (b), but only through multipliers 1 and 2 of at most ten blobs.
ALIGNED_EXISTING = ("cifar10_quick", "single_element", "not_multiple_of_4")


@pytest.mark.parametrize("name", sorted(EXISTING))
def test_mutations_a_and_b_are_invisible_on_the_old_layouts(oracle, adam, name):
    """Why the named layouts were needed: with power-of-two multipliers the operand order of Adam's rate is exact,
    and where blob ends are 4-aligned a float4 never mixes two blobs' multipliers."""
    c, lm, dm = EXISTING[name]
    got = _mutants(oracle, adam, c, lm, dm, "Adam")
    assert got["none"] is False and got["a"] is False, got
    if name in ALIGNED_EXISTING:
        assert got["b"] is False, got


# ------------------------------------------------------------- parsed multipliers

def _exact_decimal(fr, digits=70):
    q = fr.numerator * 10 ** digits // fr.denominator
    assert Fraction(q, 10 ** digits) == fr
    s = str(q).rjust(digits + 1, "0")
    return (s[:-digits] + "." + s[-digits:]).rstrip("0")


# 1 + 2^-24 + 2^-60, written out exactly: the nearest double is 1 + 2^-24, a tie between two floats that rounds to 1;
# rounded straight from the decimal to float it would be 1 + 2^-23.  protobuf's text parser reads a double and casts.
DOUBLE_ROUNDING = _exact_decimal(Fraction(1) + Fraction(1, 2 ** 24) + Fraction(1, 2 ** 60))
# (lr_mult, decay_mult) text of each blob; None: the field is absent (ParamSpec default 1)
MULTS_TEXT = [("10", "0.1"), ("0.1", None), ("0.7", "0.3"), ("20", "0"), ("3", "3"), (DOUBLE_ROUNDING, "0.1")]


def fractional_prototxt(path):
    """A solver with its net inline: three InnerProduct layers whose param specs use rounding multipliers."""
    ips = [("ip1", "data", 37), ("ip2", "ip1", 11), ("ip3", "ip2", 5)]
    layers = ['layer { name: "d" type: "Input" top: "data" input_param { shape { dim: 2 dim: 3 dim: 11 dim: 11 } } }']
    for k, (name, bottom, n) in enumerate(ips):
        specs = "".join(f" param {{ lr_mult: {lr}" + (f" decay_mult: {dm}" if dm is not None else "") + " }"
                        for lr, dm in MULTS_TEXT[2 * k:2 * k + 2])
        layers.append(f'layer {{ name: "{name}" type: "InnerProduct" bottom: "{bottom}" top: "{name}"{specs} '
                      f'inner_product_param {{ num_output: {n} }} }}')
    text = ('base_lr: 0.01\nmomentum: 0.9\nweight_decay: 0.0005\nlr_policy: "inv"\ngamma: 0.0001\npower: 0.75\n'
            'max_iter: 100\nnet_param {\n' + "\n".join(layers) + "\n}\n")
    with open(path, "w") as f:
        f.write(text)
    return str(path)


FRACTIONAL_COUNTS = [37 * 363, 37, 11 * 37, 11, 5 * 11, 5]


def expected_multipliers():
    """Per blob (lr_mult, decay_mult) as protobuf reads them: float(double(text)); an absent field is 1."""
    lm = [float(F(float(lr))) for lr, _ in MULTS_TEXT]
    dm = [float(F(float(d))) if d is not None else 1.0 for _, d in MULTS_TEXT]
    return lm, dm


def test_parsed_multipliers_round_like_protobuf(cos, tmp_path):
    d = cos.parse_solver(fractional_prototxt(tmp_path / "s.prototxt"))
    assert d.counts == FRACTIONAL_COUNTS
    lm, dm = expected_multipliers()
    assert d.lr_mult == lm and d.decay_mult == dm
    assert F(d.lr_mult[1]).tobytes() == F(0.1).tobytes() and F(d.decay_mult[0]).tobytes() == F(0.1).tobytes()
    # the double-then-float rule: 1.0, where rounding the decimal straight to float gives 1 + 2^-23
    assert d.lr_mult[-1] == 1.0
