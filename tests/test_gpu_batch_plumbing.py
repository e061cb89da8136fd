"""GPU: the batched feature calls do not synchronise with the device when their inputs are already on it.

Each call runs once under ``torch.cuda.set_sync_debug_mode("error")`` (a host synchronisation raises) on a small batch of
CUDA inputs, after its inputs and the model have been prepared outside that mode."""
import pytest
import torch

import pf_test_util as U
from oracle import weights_gen as wg
from perspectivefields_b200 import calibrate, metrics, panocam, viz

pytestmark = pytest.mark.gpu

SIZES = [(24, 32), (19, 27)]
VERSION = "Paramnet-360Cities-edina-centered"


def _fields(sizes=SIZES):
    n = len(sizes)
    return panocam.camera_fields([0.9] * n, [h for h, _ in sizes], [w for _, w in sizes], [-0.2] * n, [0.1] * n, [0.02] * n, [-0.01] * n)


def _results():
    ups, lats = _fields()
    return [{"pred_gravity_original": u.permute(2, 0, 1), "pred_latitude_original": l} for u, l in zip(ups, lats)], ups, lats


def _camera_fields():
    return lambda: _fields()


def _crop_distortion_views():
    pano = torch.from_numpy(wg.smooth_images(1, 64, 128, seed=1)[0]).cuda()
    return lambda: panocam.crop_distortion_views(pano, [(60.0, 0.0, 24, 32, 10.0, -5.0, 3.0), (45.0, 0.2, 19, 27, 80.0, 12.0, -4.0)])


def _crop_equi_views():
    pano = torch.from_numpy(wg.smooth_images(1, 64, 128, seed=2)[0]).cuda()
    return lambda: panocam.crop_equi_views(pano, [(60.0, 32, 24, 10.0, -5.0, 3.0, 4 / 3), (70.0, 27, 19, 80.0, 0.0, -4.0, 1.0)])


def _draw_fields_batch():
    imgs = [torch.from_numpy(wg.smooth_images(1, h, w, seed=3)[0]).cuda() for h, w in SIZES]
    ups, lats = _fields()
    lats = [torch.deg2rad(l) for l in lats]
    return lambda: viz.draw_fields_batch(imgs, ups, lats, density=4)


def _field_errors():
    res, ups, lats = _results()
    return lambda: metrics.field_errors(res, ups, lats, return_maps=True)


def _fit_camera():
    res, _, _ = _results()
    return lambda: calibrate.fit_camera(res, init="fields", max_iterations=5)


def _model_and_fields():
    m = U.make_model(VERSION, seed=0, device="cuda")[0]
    h, w = m.net_size()
    ups, lats = _fields([(h, w)] * 2)
    return m, ups, lats


def _targets_from_fields():
    m, ups, lats = _model_and_fields()
    return lambda: m.targets_from_fields(ups, lats)


def _losses():
    m, ups, lats = _model_and_fields()
    res = m.inference_batch(wg.smooth_images(2, *m.net_size(), seed=5))
    tg = m.targets_from_fields(ups, lats)
    return lambda: m.losses(res, tg)


CALLS = {"camera_fields": _camera_fields, "crop_distortion_views": _crop_distortion_views, "crop_equi_views": _crop_equi_views,
         "draw_fields_batch": _draw_fields_batch, "field_errors": _field_errors, "fit_camera": _fit_camera,
         "targets_from_fields": _targets_from_fields, "losses": _losses}


@pytest.mark.parametrize("call", list(CALLS))
def test_calls_on_device_inputs_do_not_synchronise(call):
    run = CALLS[call]()
    run()                                    # first call: module loads and allocator growth happen outside the checked window
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        run()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
