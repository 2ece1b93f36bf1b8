"""The bounds of tests/net_harness.py on the oracles' own outputs: check_float16 and check_float32 pass them as they are
and fail each perturbation just past a bound; the bit checks fail one changed bit; expected_launches gives the launch
counts of the layer plans the per-family launch tests were written with."""
import numpy as np
import pytest

from tests import net_harness as nh


@pytest.fixture(scope="module")
def oracle_out():
    """-> (Out of the oracle's own outputs, the oracle's outputs) of RISEv3.3, which has the WDL / plies outputs"""
    kind = nh.KINDS["risev33"]
    arch = kind.arch()
    ref = kind.forward(kind.weights(arch), arch, nh.inputs(arch, 4, 5))
    return nh.Out(ref["value"].copy(), ref["prob"].copy(), ref["aux"].copy()), ref


def _value(out, bound):
    out.value[1] += 1.1 * bound


def _prob(out, rtol):
    out.prob[2, out.prob[2].argmax()] *= 1 + 1.1 * rtol


def _aux(out, bound):
    out.aux[3, 0] += 1.1 * bound


def _row_sum(out, _):
    out.prob[0] *= 1 + 1.1 * nh.PROB_SUM_ATOL  # every ratio, and so the centred logits, unchanged


def _logit(out, bound):
    """a probability near 1e-4 scaled by exp(1.1 bound): within its rtol, and too small to move the row's sum"""
    out.prob[1, np.abs(np.log(out.prob[1] / 1e-4)).argmin()] *= np.exp(1.1 * bound)


# precision: (check, {perturbation: (bound, what the failure names)})
CHECKS = {"float16": (nh.check_float16, {"value": (nh.VALUE_ATOL, "value"), "prob": (nh.PROB_RTOL, "probabilities"),
                                         "aux": (nh.AUX_ATOL, "aux"), "row_sum": (None, "probability row sums"),
                                         "logit": (nh.LOGIT_ATOL, "centred logits")}),
          "float32": (nh.check_float32, {"value": (nh.F32_ATOL, "value"), "prob": (nh.F32_PROB_RTOL, "probabilities"),
                                         "aux": (nh.F32_ATOL, "aux"), "row_sum": (None, "probability row sums"),
                                         "logit": (nh.F32_LOGIT_ATOL, "centred logits")})}
PERTURB = {"value": _value, "prob": _prob, "aux": _aux, "row_sum": _row_sum, "logit": _logit}


@pytest.mark.parametrize("precision", sorted(CHECKS))
def test_checks_pass_the_oracles_own_outputs(oracle_out, precision):
    out, ref = oracle_out
    CHECKS[precision][0](out, ref)


@pytest.mark.parametrize("what", sorted(PERTURB))
@pytest.mark.parametrize("precision", sorted(CHECKS))
def test_checks_fail_just_past_each_bound(oracle_out, precision, what):
    """each perturbation fails the check of the bound it passes"""
    check, bounds = CHECKS[precision]
    bound, name = bounds[what]
    out, ref = oracle_out
    out = nh.Out(*(t.copy() for t in out))
    PERTURB[what](out, bound)
    with pytest.raises(AssertionError, match=name):
        check(out, ref)


@pytest.mark.parametrize("field", nh.Out._fields)
def test_same_bits_fails_one_changed_bit(oracle_out, field):
    out, _ = oracle_out
    changed = nh.Out(*(t.copy() for t in out))
    getattr(changed, field).view(np.uint32).flat[0] ^= 1
    assert nh.same_bits(out, nh.Out(*(t.copy() for t in out))) and not nh.same_bits(out, changed)


def test_expected_launches_reproduce_the_family_formulas():
    def tower(arch, precision):  # the per-family tests' tower: one kernel (float16) or 3 launches per block + SE
        return 1 if precision == "float16" else sum(3 + (se is not None) for se in arch["se_types"])

    for precision in ("float16", "float32"):
        for kind in ("risev33", "mx_risev2"):  # input conversion, stem, tower, value head, two policy convs, softmax
            a = nh.KINDS[kind].arch()
            assert nh.expected_launches(a, precision) == 1 + 1 + tower(a, precision) + 4, kind
        a = nh.KINDS["fc_risev33_76_1968"].arch()  # ... and the fully-connected layer
        assert nh.expected_launches(a, precision) == 1 + 1 + tower(a, precision) + 5
        a = nh.KINDS["av_normal"].arch()  # per NTB 9 launches in float16 (10 in float32), one tower launch per segment
        segments = 1 + sum(1 for i, t in enumerate(a["ntb"][:-1]) if t and not a["ntb"][i + 1])
        n_ntb, n_plain = sum(a["ntb"]), len(a["ntb"]) - sum(a["ntb"])
        assert nh.expected_launches(a, precision) == 1 + 1 + 4 + (
            segments + 9 * n_ntb if precision == "float16" else 3 * n_plain + 10 * n_ntb)
    # the geometry rows' counts, which their launch test holds the device to
    counts = {"av_small": (16, 79), "av_large": (26, 131), "narrow64": (17, 25), "full256_ntb": (25, 32),
              "mid160": (17, 25), "heads_max": (7, 12), "heads_min": (7, 9), "rise25": (8, 90), "rise49": (9, 170),
              "av_long_run": (18, 97)}
    assert sorted(counts) == sorted(nh.GEOMETRIES)
    for name, (f16, f32) in counts.items():
        a = nh.KINDS[name].arch()
        assert (nh.expected_launches(a, "float16"), nh.expected_launches(a, "float32")) == (f16, f32), name
