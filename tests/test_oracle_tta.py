"""CPU: properties of the flip test-time augmentation rule as tests/oracle_tta.py states it (DESIGN.md section 1, "Flip test-time
augmentation"): the up head's class map is the mirror of the bin directions, and the merges are exactly mirror-equivariant."""
import numpy as np
import pytest
import torch

import oracle_tta as ot
from oracle import model as om

F32 = np.float32


def test_class_map_is_the_mirror_of_the_bin_directions():
    P = ot.class_map(73, True)
    assert np.array_equal(P[P], np.arange(73))                    # an involution
    for c in (18, 54, 72):                                        # straight up, straight down, no direction
        assert P[c] == c
    assert sorted(set(P.tolist())) == list(range(73))
    vec = om.decode_bin(torch.arange(73), 73).numpy()             # [2, 73] bin-centre directions (bin 72: zero)
    mirrored = vec[:, P]
    assert np.abs(mirrored[0] + vec[0]).max() < 1e-6              # x negated ...
    assert np.abs(mirrored[1] - vec[1]).max() < 1e-6              # ... y kept
    assert np.array_equal(ot.class_map(180, False), np.arange(180))


def _pairs(shape, seed):
    g = np.random.default_rng(seed)
    return g.standard_normal(shape).astype(F32), g.standard_normal(shape).astype(F32)


def _unit(v):
    return (v / np.linalg.norm(v, axis=-3, keepdims=True)).astype(F32)


@pytest.mark.parametrize("W", [8, 7])
def test_merge_of_the_mirror_is_the_mirror_of_the_merge(W):
    """Swapping the image and its mirror (the merge of x~) gives the mirror of merge(x): for the up vectors with x negated, for
    the logits with the classes mapped -- exactly, bit for bit."""
    a, b = _pairs((3, 2, 5, W), 1)
    a, b = _unit(a), _unit(b)
    m, mt = ot.merge_up(a, b), ot.merge_up(b, a)
    assert np.array_equal(mt[:, 0], -ot.mirror(m[:, 0])) and np.array_equal(mt[:, 1], ot.mirror(m[:, 1]))
    la, lb = _pairs((3, 5, W), 2)
    assert np.array_equal(ot.merge_lat(lb, la), ot.mirror(ot.merge_lat(la, lb)))
    for nc, grav in ((73, True), (180, False)):
        ga, gb = _pairs((2, nc, 4, W), nc)
        P = ot.class_map(nc, grav)
        want = np.take(ot.mirror(ot.merge_logits(ga, gb, grav)), P, axis=-3)
        assert np.array_equal(ot.merge_logits(gb, ga, grav), want)


def test_symmetric_input_gives_antisymmetric_up_x_and_symmetric_latitude():
    """x == x~: both slots hold the same outputs, so the merge leaves up_x antisymmetric and up_y, the latitude and (with the
    class map) the logits symmetric about the centre column, exactly."""
    a, _ = _pairs((2, 2, 6, 9), 3)
    a = _unit(a)
    m = ot.merge_up(a, a)
    assert np.array_equal(m[:, 0], -ot.mirror(m[:, 0])) and np.array_equal(m[:, 1], ot.mirror(m[:, 1]))
    assert np.all(m[:, 0, :, 4] == 0)                              # the centre column of an odd width
    l, _ = _pairs((2, 6, 9), 4)
    ml = ot.merge_lat(l, l)
    assert np.array_equal(ml, ot.mirror(ml))
    g, _ = _pairs((1, 73, 3, 9), 5)
    mg = ot.merge_logits(g, g, True)
    assert np.array_equal(mg, np.take(ot.mirror(mg), ot.class_map(73, True), axis=-3))


def test_merge_is_a_sum_then_a_scale():
    a, b = _pairs((1, 4, 3), 6)
    assert np.array_equal(ot.merge_lat(a, b), (a + ot.mirror(b)) * F32(0.5))
    u = ot.merge_up(np.zeros((1, 2, 1, 2), F32), np.zeros((1, 2, 1, 2), F32))
    assert np.array_equal(u, np.zeros_like(u))                     # normalize(0) = 0 (max(|v|, 1e-12))
