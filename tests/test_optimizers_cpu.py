"""CPU tests of the OPTIMIZER cfg switch (no GPU needed): the cfg table, the C enum against the binding, and first steps of the
float32 optimizer oracle against values worked out by hand in float64."""
import configparser
import os
import re

import numpy as np
import pytest

from oracle import optimizer_oracle as OO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

EXPECTED = {   # cfg name -> (aae_optimizer_kind, hp at TF's defaults, slot names)
    "Adam": (0, (0.9, 0.999, 1e-8), ("Adam", "Adam_1")),
    "GradientDescent": (1, (), ()),
    "ProximalGradientDescent": (1, (), ()),
    "Adagrad": (2, (0.1,), ("Adagrad",)),
    "ProximalAdagrad": (3, (0.1,), ("ProximalAdagrad",)),
    "Adadelta": (4, (0.95, 1e-8), ("Adadelta", "Adadelta_1")),
    "RMSProp": (5, (0.9, 0.0, 1e-10), ("RMSProp", "RMSProp_1")),
    "Ftrl": (6, (0.1,), ("Ftrl", "Ftrl_1")),
}


def _args(name):
    c = configparser.ConfigParser()
    c.read_dict({"Training": {"BATCH_SIZE": "4", "LEARNING_RATE": "2e-4", "OPTIMIZER": name}})
    return c


@pytest.mark.parametrize("name", sorted(EXPECTED))
def test_cfg_names_give_kind_hp_and_slots(name):
    from augmentedautoencoder_b200.ae import ae_factory as F
    kind, hp, slots = EXPECTED[name]
    assert F.OPTIMIZERS[name] == EXPECTED[name]
    top = F.build_train_op(object(), _args(name))      # no trainer is created before the first step
    assert top._opt.kind == kind and top._slots == slots
    assert np.float32(top._opt.learning_rate) == np.float32(2e-4)
    assert list(top._opt.hp) == [float(np.float32(v)) for v in hp] + [0.0] * (4 - len(hp))


@pytest.mark.parametrize("name,needs", [("Momentum", "momentum"), ("AdagradDA", "global_step")])
def test_optimizers_the_reference_cannot_build_from_a_cfg_are_refused(name, needs):
    from augmentedautoencoder_b200.ae import ae_factory as F
    with pytest.raises(ValueError, match="needs `%s`.*reference cannot build it from a cfg either" % needs):
        F.build_train_op(object(), _args(name))


def test_unknown_optimizer_is_refused_naming_the_supported_set():
    from augmentedautoencoder_b200.ae import ae_factory as F
    with pytest.raises(ValueError, match="Foo") as e:
        F.build_train_op(object(), _args("Foo"))
    assert all(n in str(e.value) for n in EXPECTED)
    with pytest.raises(ValueError, match="Foo"):
        F.TrainOp(object(), 2e-4, optimizer="Foo")


def test_header_and_binding_agree_on_the_optimizer_kinds():
    from augmentedautoencoder_b200 import _lib
    src = open(os.path.join(ROOT, "include", "aae_b200.h")).read()
    body = re.search(r"typedef enum \{([^}]*)\} aae_optimizer_kind;", src).group(1)
    kinds = {k: int(v) for k, v in re.findall(r"AAE_OPT_(\w+)\s*=\s*(\d+)", body)}
    assert kinds == {"ADAM": 0, "GRADIENT_DESCENT": 1, "ADAGRAD": 2, "PROXIMAL_ADAGRAD": 3, "ADADELTA": 4, "RMSPROP": 5, "FTRL": 6}
    assert {k: getattr(_lib, "OPT_" + k) for k in kinds} == kinds
    assert set(OO.RULES) == set(kinds.values()) - {0}
    assert re.search(r"typedef struct \{\s*int32_t kind;[^}]*float learning_rate;\s*float hp\[4\];\s*\} aae_optimizer;", src)
    assert [f[0] for f in _lib.Optimizer._fields_] == ["kind", "learning_rate", "hp"]


f32 = np.float32
P = np.array([0.5, -0.25, 0.125, 0.0, 1.5], f32)
G = np.array([0.5, 0.75, -0.3, 0.0, -2.0], f32)
LR = 0.01


def _near(got, want64, ulps=4):
    assert got.dtype == np.float32
    want = np.asarray(want64, np.float64)
    assert np.all(np.abs(got - want) <= ulps * np.spacing(np.abs(want).astype(f32)) + 1e-30), (got, want)


def test_rmsprop_first_step_from_rms_one():
    p, (ms, mom) = OO.rmsprop(P, G, (np.ones_like(P), np.zeros_like(P)), LR)
    g, p0 = G.astype(np.float64), P.astype(np.float64)
    ms64 = 1.0 + (g * g - 1.0) * 0.1
    mom64 = (g * LR) / np.sqrt(ms64 + 1e-10)
    _near(ms, ms64)
    _near(mom, mom64)
    _near(p, p0 - mom64)
    assert mom[3] == 0 and p[3] == P[3]


def test_adagrad_first_step_from_initial_accumulator():
    p, (acc,) = OO.adagrad(P, G, (np.full_like(P, 0.1),), LR)
    g = G.astype(np.float64)
    acc64 = 0.1 + g * g
    _near(acc, acc64)
    _near(p, P - g * LR / np.sqrt(acc64))


def test_adadelta_first_step_from_zero_state():
    z = np.zeros_like(P)
    p, (acc, accu) = OO.adadelta(P, G, (z, z), LR)
    g = G.astype(np.float64)
    acc64 = g * g * 0.05
    upd = np.sqrt(1e-8) / np.sqrt(acc64 + 1e-8) * g
    _near(acc, acc64)
    _near(p, P - upd * LR)
    _near(accu, upd * upd * 0.05, ulps=8)


def test_ftrl_first_step_both_signs_of_linear():
    acc0 = np.full_like(P, 0.1)
    p, (acc, lin) = OO.ftrl(P, G, (acc0, np.zeros_like(P)), LR)
    g, p0 = G.astype(np.float64), P.astype(np.float64)
    new = 0.1 + g * g
    lin64 = g - ((np.sqrt(new) - np.sqrt(0.1)) / LR) * p0
    assert (lin64 > 0).any() and (lin64 < 0).any()
    _near(acc, new)
    _near(lin, lin64, ulps=16)
    want = np.where(np.abs(lin64) > 0, -lin64 / (np.sqrt(new) / LR), 0.0)
    _near(p, want, ulps=16)
    assert lin[3] == 0 and p[3] == 0          # |linear| = 0 is not > l1 = 0: the weight is set to 0


def test_proximal_gradient_descent_is_gradient_descent_bit_for_bit():
    rng = np.random.RandomState(0)
    p, g = rng.standard_normal(100000).astype(f32), rng.standard_normal(100000).astype(f32)
    a, _ = OO.gradient_descent(p, g, (), 2e-4)
    b, _ = OO.proximal_gradient_descent(p, g, (), 2e-4)
    assert np.array_equal(a, b)


def test_proximal_adagrad_rounds_differently_from_adagrad():
    rng = np.random.RandomState(1)
    p, g = rng.standard_normal(100000).astype(f32), rng.standard_normal(100000).astype(f32)
    acc = np.full_like(p, 0.1)
    a, (sa,) = OO.adagrad(p, g, (acc,), 2e-4)
    b, (sb,) = OO.proximal_adagrad(p, g, (acc,), 2e-4)
    assert np.array_equal(sa, sb)
    step_a, step_b = (p - a).astype(np.float64), (p - b).astype(np.float64)
    # the same value to rounding: the two products differ by at most an ulp or two of the step, then one more rounding of the difference
    tol = np.spacing(np.maximum(np.abs(a), np.abs(b))).astype(np.float64) + 2.0 ** -22 * np.abs(step_a)
    assert np.all(np.abs(a.astype(np.float64) - b) <= tol)
    assert not np.array_equal(a, b) and np.abs(step_a - step_b).max() > 0


def _round_f32(x):
    """the float32 nearest to the rational x, ties to the even significand"""
    from fractions import Fraction
    r = np.float32(float(x))
    cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
    return min(cands, key=lambda c: (abs(Fraction(float(c)) - x), int(np.array(c).view(np.uint32)) & 1))


def test_fma32_rounds_once():
    """OO.fma32 (the kernel's Adam FMAs in the replay) against the exact product-sum rounded once, on random operands of mixed
    magnitude and on a constructed case where the float64 sum lands on a float32 midpoint: there the sum rounded twice is one ulp
    off and fma32 is not."""
    from fractions import Fraction
    rng = np.random.RandomState(0)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.randint(-30, 10, n)).astype(np.float32)
    b = (rng.standard_normal(n) * 2.0 ** rng.randint(-30, 10, n)).astype(np.float32)
    c = (rng.standard_normal(n) * 2.0 ** rng.randint(-40, 10, n)).astype(np.float32)
    got = OO.fma32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got, want)
    u = 2.0 ** -23
    a, b, c = np.float32(1 + u), np.float32((1 - u) * 2.0 ** -24), np.float32(1 + u)     # a b + c = 1 + u + u/2 - 2^-70
    exact = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    assert OO.fma32(a, b, c) == np.float32(1 + u) == _round_f32(exact)
    assert np.float32(np.float64(a) * np.float64(b) + np.float64(c)) == np.float32(1 + 2 * u)    # rounded twice
