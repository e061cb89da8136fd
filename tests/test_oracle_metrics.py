"""CPU: the scoring oracle (tests/oracle_metrics.py) against the unmodified reference's encoders and head losses
(tests/golden/losses.npz), and the targets rule against the inference decode it inverts."""
import math
import os

import numpy as np
import pytest
import torch

import oracle_metrics as om

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "losses.npz"))


def test_encode_bin_matches_reference_on_centres_zeros_and_ties():
    v, ties = om.special_vectors()
    assert ties >= 60
    assert np.array_equal(om.encode_bin(v, om.NUM_BIN).numpy(), G["enc_special"].astype(np.int64))


def test_encode_bin_latitude_matches_reference_on_boundaries():
    b = om.latitude_boundaries(om.NUM_LAT)
    lat = np.concatenate([b, np.nextafter(b, np.float32(-np.inf)), np.nextafter(b, np.float32(np.inf)),
                          np.array([-90.0, 90.0, -89.99, 89.99, 0.0, -0.0, -100.0, 100.0], np.float32)]).astype(np.float32)
    assert np.array_equal(om.encode_bin_latitude(lat, om.NUM_LAT).numpy(), G["enc_lat_special"].astype(np.int64))


def test_msgil_norm_loss_matches_reference():
    g = torch.Generator().manual_seed(3)
    p, t = torch.randn((2, 2, 37, 53), generator=g), torch.randn((2, 2, 37, 53), generator=g)
    mask = torch.rand((2, 2, 37, 53), generator=g) < 0.7
    assert om._msg(p.double() - t.double(), mask) == pytest.approx(float(G["msgil"]), rel=1e-6)


@pytest.mark.parametrize("case", om.LOSS_CASES, ids=[c[0] for c in om.LOSS_CASES])
def test_losses_match_reference(case):
    name, loss_type, n, h, w, seed = case
    pg, pl, up, lat = om.loss_inputs(loss_type, n, h, w, seed)
    gg, gl = om.targets(up, lat, loss_type)
    if loss_type == "classification":
        assert om.label_checksum(gg) == int(G[name + "/gt_gravity_checksum"])
        assert om.label_checksum(gl) == int(G[name + "/gt_latitude_checksum"])
        assert bool((gg == om.IGNORE_GRAVITY).any())   # the invalid (zero) vectors are ignored
    else:
        assert bool((up == 0).all(-1).any())
    got = om.losses(pg, pl, gg, gl, loss_type)
    keys = [k[len(name) + 1:] for k in G.files if k.startswith(name + "/") and not k.endswith("_checksum")]
    assert sorted(keys) == sorted(got)
    for k in keys:
        assert got[k] == pytest.approx(float(G[f"{name}/{k}"]), rel=1e-6), k


def test_no_valid_pixel_gives_nan():
    """Where the reference stops in pdb: the gravity L2 term over no valid target, a cross-entropy with every label ignored."""
    pg, pl, up, lat = om.loss_inputs("regression", 1, 64, 64, 1)
    gg, gl = om.targets(torch.zeros_like(up), lat, "regression")
    got = om.losses(pg, pl, gg, gl, "regression")
    assert math.isnan(got["gravity-l2-loss"]) and got["gravity-msg-normal-loss"] == 0.0
    pg, pl, up, lat = om.loss_inputs("classification", 1, 32, 32, 1)
    gg, gl = om.targets(torch.zeros_like(up), lat, "classification")
    assert math.isnan(om.losses(pg, pl, gg, gl, "classification")["loss_gravity"])


def test_targets_rule_round_trips_through_the_decode():
    g = torch.Generator().manual_seed(7)
    up = om.random_up(g, 2, 40, 56)
    lat = om.random_lat_deg(g, 2, 40, 56)
    gg, gl = om.targets(up, lat, "classification")
    for b in range(2):
        dec = om.decode_bin(gg[b], om.NUM_BIN)
        u = up[b].permute(2, 0, 1).double()
        valid = (u != 0).any(0)
        assert bool((gg[b][~valid] == om.NUM_BIN - 1).all())
        ang = torch.rad2deg(torch.atan2(dec[0] * u[1] - dec[1] * u[0], (dec * u).sum(0)).abs())
        assert float(ang[valid].max()) <= 2.5 + 1e-4          # within half a bin (5 degrees wide)
    half = 180 / om.NUM_LAT / 2
    centres = -90 + (gl.double() + 0.5) * (180 / om.NUM_LAT)
    assert float((centres - lat.double()).abs().max()) <= half + 1e-4
    rg, rl = om.targets(up, lat, "regression")
    assert torch.equal(rg, up.permute(0, 3, 1, 2))
    # float32 sin: asin's slope near +-90 turns one ulp of sin (6e-8) into up to sqrt(2 * 6e-8) rad = 0.02 degrees
    assert float((torch.rad2deg(torch.asin(rl[:, 0].double())) - lat.double()).abs().max()) < 0.03
    assert float((torch.rad2deg(torch.asin(rl[:, 0].double())) - lat.double())[lat.abs() < 80].abs().max()) < 1e-4
    _, rl_rad = om.targets(up, torch.deg2rad(lat), "regression", lat_mode="rad")
    assert float((rl_rad - rl).abs().max()) < 1e-6


def test_field_error_rule():
    pu = np.array([[[1.0, 0.0, 0.0, 1e-6, 1.0]], [[0.0, 1.0, 0.0, 0.0, 0.0]]])            # [2, 1, 5]
    gu = np.array([[[0.0, 2.0], [0.0, 1.0], [1.0, 0.0], [1.0, 1.0], [0.0, 1e-6]]])         # [1, 5, 2]
    eu, el = om.error_maps(pu, np.array([[10.0, 0.0, np.nan, 5.0, 0.0]]), gu, np.array([[0.0, np.nan, 1.0, -5.0, 0.0]]))
    assert np.allclose(eu, [[90.0, 0.0, 180.0, 180.0, np.nan]], equal_nan=True)
    assert np.allclose(el, [[10.0, np.nan, np.inf, 10.0, 0.0]], equal_nan=True)
    c, mean, med, fr = om.stats(np.array([3.0, np.nan, 1.0, 2.0, 10.0]), (2.0, 5.0))
    assert (c, mean, med, fr) == (4, 4.0, 2.5, [0.25, 0.75])
    assert om.stats(np.array([np.nan]), (1.0,))[0] == 0
