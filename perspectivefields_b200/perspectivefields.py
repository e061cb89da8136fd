"""Drop-in for ``perspective2d.PerspectiveFields`` (reference: perspective2d/perspectivefields.py:121-272) whose
whole forward runs in libpf_b200.so (hand-written sm_90a CUDA, C ABI in include/pf_b200.h).

Kept from the reference surface: ``PerspectiveFields(version)``, ``.eval()``, ``.cuda()/.to()``, ``.device``,
``.versions()``, ``.inference(img_bgr)``, ``.inference_batch(list)``, ``.forward(batched_inputs)``, ``.param_net(predictions)``,
``.state_dict()/.load_state_dict()`` with the reference's key names, attributes ``version``, ``param_on``, ``cfg``,
``input_format``; result dictionaries with the same keys, order, shapes and dtypes.  There is no CPU path: the model
must live on a CUDA device (H100) and libpf_b200.so must be built, otherwise inference raises.
"""
import collections
import ctypes
import itertools

import numpy as np
import torch
from torch import nn

from . import _batch, _native
from .checkpoint import checkpoint_schema, default_state, load_zoo_checkpoint
from .variants import PIXEL_MEAN, PIXEL_STD, RESIZE, VARIANTS, make_cfg, model_zoo
from .weights import PN, param_net_grad_to_ref, param_net_train_weights, repack, repack_param_net

_ENGINE_SERIAL = itertools.count()


def check_resize(resize):
    """``PerspectiveFields(resize=...)`` -> the working size (H, W).  ``None``: the yaml's DATALOADER.RESIZE ([320, 320]).  H and W
    (the reference's [Height, Width] order) must be multiples of 32 in [64, 640] with (H/32) * (W/32) <= 256: the attention key
    count of every MiT stage (100 at 320 x 320); 64 keeps the smallest head level at 2 x 2 or more."""
    if resize is None:
        return tuple(int(x) for x in RESIZE)
    try:
        h, w = resize
    except (TypeError, ValueError):
        raise ValueError(f"resize must be None or (height, width), got {resize!r}") from None
    if not all(isinstance(x, (int, np.integer)) and not isinstance(x, bool) for x in (h, w)):
        raise ValueError(f"resize must hold two integers, got {resize!r}")
    h, w = int(h), int(w)
    if h % 32 or w % 32 or not (64 <= h <= 640 and 64 <= w <= 640):
        raise ValueError(f"resize {(h, w)}: height and width must be multiples of 32 in [64, 640]")
    if (h // 32) * (w // 32) > 256:
        raise ValueError(f"resize {(h, w)}: (H/32) * (W/32) = {(h // 32) * (w // 32)} attention keys, at most 256 are supported")
    return h, w


class _Engine:
    """One libpf_b200 handle + its device-resident repacked weights and scratch, for one CUDA device."""

    def __init__(self, device, version, ref_state, net_hw=RESIZE):
        self.L = _native.lib()
        self.device = device
        cfg = VARIANTS[version]
        desc = _native.pf_model_desc()
        desc.gravity_classes, desc.latitude_classes = cfg["gravity_classes"], cfg["latitude_classes"]
        desc.param_net = {None: _native.PF_PARAM_NONE, "ParamNet": _native.PF_PARAM_CENTERED,
                          "ParamNetConvNextRegress": _native.PF_PARAM_UNCENTERED}[cfg["param_net"]]
        desc.param_input_size = cfg["input_size"]
        desc.pixel_mean[:] = PIXEL_MEAN
        desc.pixel_std[:] = PIXEL_STD
        self.net_h, self.net_w = int(net_hw[0]), int(net_hw[1])
        self.handle = ctypes.c_void_p()
        if (self.net_h, self.net_w) == tuple(RESIZE):
            _native.check(self.L.pf_create(device.index, ctypes.byref(desc), ctypes.byref(self.handle)))
        else:
            _native.check(self.L.pf_create_sized(device.index, ctypes.byref(desc), self.net_h, self.net_w, ctypes.byref(self.handle)))
        self.tensors = {}
        for name, t in repack(ref_state, cfg).items():
            d = t.to(device)
            self.tensors[name] = d  # keeps the device memory alive for the lifetime of the handle
            dt = _native.PF_BF16 if d.dtype == torch.bfloat16 else _native.PF_F32
            _native.check(self.L.pf_set_weight(self.handle, name.encode(), d.data_ptr(), d.numel(), dt))
        _native.check(self.L.pf_finalize(self.handle))
        self.workspace = None
        self.ws_stream = None      # stream of the last forward that used the workspace
        self.ws_event = None       # ... and its completion
        self.decode_only = False
        self.confidence = False      # pf_forward_confidence: the head-confidence maps as well
        self.pinned = None
        self.pinned_event = None
        self.dev_blob = None
        self.staged_slot = None
        self.serial = next(_ENGINE_SERIAL)
        self.train_ready = False     # the backward's extra ParamNet tensors are registered (register_train_weights)
        self._grad_layout = None

    def register_train_weights(self, tensors):
        """Registers ParamNet's backward-only tensors (weights.param_net_train_weights, already on the device) with the engine."""
        for name, d in tensors.items():
            self.tensors[name] = d
            dt = _native.PF_BF16 if d.dtype == torch.bfloat16 else _native.PF_F32
            _native.check(self.L.pf_set_weight(self.handle, name.encode(), d.data_ptr(), d.numel(), dt))
        _native.check(self.L.pf_finalize(self.handle))
        self.train_ready = True

    def grad_layout(self):
        """[(engine weight name, offset, numel)] of pf_param_backward's gradient buffer."""
        if self._grad_layout is None:
            out, total, i = [], int(self.L.pf_param_grad_numel()), 0
            name, off, num = ctypes.c_char_p(), ctypes.c_int64(), ctypes.c_int64()
            while not out or out[-1][1] + out[-1][2] < total:
                _native.check(self.L.pf_param_grad_entry(i, ctypes.byref(name), ctypes.byref(off), ctypes.byref(num)))
                out.append((name.value.decode(), off.value, num.value))
                i += 1
            self._grad_layout = out
        return self._grad_layout

    def close(self):
        if self.handle:
            self.L.pf_destroy(self.handle)
            self.handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _workspace(self, need, cur):
        """Scratch of ``need`` bytes for pf_forward / pf_param_forward.  The buffer is allocated from torch's caching allocator on
        the stream of its first use; a caller that switches streams between calls is kept safe by stream-ordering the hand-over:
        the new stream waits for the last call that used the workspace (``ws_event``), and a workspace that is replaced is marked
        as used by that stream (``record_stream``) so that its block is not recycled under a call still running there."""
        if self.ws_event is not None and self.ws_stream is not None and self.ws_stream != cur:
            cur.wait_event(self.ws_event)
        if self.workspace is None or self.workspace.numel() < need:
            if self.workspace is not None and self.ws_stream is not None:
                self.workspace.record_stream(self.ws_stream)
            self.workspace = None
            self.workspace = torch.empty(need, dtype=torch.uint8, device=self.device)
        self.ws_stream = cur
        return self.workspace

    def stage_images(self, imgs):
        """Host uint8 images -> one pinned blob -> one async H2D copy on a dedicated copy stream (two pinned / device blob pairs,
        so the upload of batch k+1 overlaps the forward of batch k).  Returns (device blob, offsets); the current stream has been
        made to wait for the upload."""
        sizes = [im.size for im in imgs]
        offsets = np.zeros(len(imgs), np.int64)
        np.cumsum(sizes[:-1], out=offsets[1:])
        total = int(sum(sizes))
        if self.pinned is None or self.pinned[0].numel() < total:
            cap = max(total, 1 << 20)
            self.pinned = [torch.empty(cap, dtype=torch.uint8).pin_memory() for _ in range(2)]
            self.dev_blob = [torch.empty(cap, dtype=torch.uint8, device=self.device) for _ in range(2)]
            self.pinned_event = [None, None]    # upload from pinned[s] has completed
            self.blob_free = [None, None]       # the forward that read dev_blob[s] has completed (recorded by forward())
            self.h2d_stream = torch.cuda.Stream(device=self.device)
            self.slot = 0
        s = self.slot = self.slot ^ 1
        if self.pinned_event[s] is not None:
            self.pinned_event[s].synchronize()  # the upload that last used this pinned buffer must have drained before it is rewritten
        host = self.pinned[s].numpy()
        for im, off in zip(imgs, offsets):
            host[off:off + im.size] = im.reshape(-1)
        cur = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.h2d_stream):
            if self.blob_free[s] is not None:
                self.h2d_stream.wait_event(self.blob_free[s])
            else:
                self.h2d_stream.wait_stream(cur)
            self.dev_blob[s][:total].copy_(self.pinned[s][:total], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record(self.h2d_stream)
        self.pinned_event[s] = ev
        cur.wait_event(ev)
        self.staged_slot = s
        return self.dev_blob[s], offsets

    def forward(self, n, heights, widths, blob=None, offsets=None, chw=None):
        dev = self.device
        h = np.ascontiguousarray(heights, np.int32)
        w = np.ascontiguousarray(widths, np.int32)
        hw = h.astype(np.int64) * w.astype(np.int64)
        g_off = np.zeros(n, np.int64)
        l_off = np.zeros(n, np.int64)
        np.cumsum(2 * hw[:-1], out=g_off[1:])
        np.cumsum(hw[:-1], out=l_off[1:])
        cur = torch.cuda.current_stream(dev)
        gc_, lc_ = (2, 1) if self.decode_only else (self.gravity_classes, self.latitude_classes)
        out = {
            "pred_gravity": torch.empty((n, gc_, self.net_h, self.net_w), dtype=torch.float32, device=dev),
            "pred_latitude": torch.empty((n, lc_, self.net_h, self.net_w), dtype=torch.float32, device=dev),
            "gravity_original": torch.empty(int(2 * hw.sum()), dtype=torch.float32, device=dev),
            "latitude_original": torch.empty(int(hw.sum()), dtype=torch.float32, device=dev),
            "params": torch.empty((n, 8), dtype=torch.float32, device=dev),
            "g_off": g_off, "l_off": l_off, "h": h, "w": w,
        }
        if self.confidence:
            for k in ("gravity_confidence", "latitude_confidence"):
                out[k] = torch.empty((n, self.net_h, self.net_w), dtype=torch.float32, device=dev)
                out[k + "_original"] = torch.empty(int(hw.sum()), dtype=torch.float32, device=dev)
        ws = self._workspace(_native.check(self.L.pf_workspace_bytes(self.handle, n, int(h.max()))), cur)
        bt = _native.pf_batch()
        bt.n = n
        i64p, i32p = ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int32)
        if blob is not None:
            offsets = np.ascontiguousarray(offsets, np.int64)
            bt.images_u8 = blob.data_ptr()
            bt.image_offset = offsets.ctypes.data_as(i64p)
        else:
            bt.images_chw = chw.data_ptr()
        bt.height, bt.width = h.ctypes.data_as(i32p), w.ctypes.data_as(i32p)
        bt.pred_gravity, bt.pred_latitude = out["pred_gravity"].data_ptr(), out["pred_latitude"].data_ptr()
        bt.gravity_original, bt.gravity_original_offset = out["gravity_original"].data_ptr(), g_off.ctypes.data_as(i64p)
        bt.latitude_original, bt.latitude_original_offset = out["latitude_original"].data_ptr(), l_off.ctypes.data_as(i64p)
        bt.params = out["params"].data_ptr()
        if self.confidence:
            cf = _native.pf_confidence(out["gravity_confidence"].data_ptr(), out["latitude_confidence"].data_ptr(),
                                       out["gravity_confidence_original"].data_ptr(), out["latitude_confidence_original"].data_ptr())
            _native.check(self.L.pf_forward_confidence(self.handle, ctypes.byref(bt), ctypes.byref(cf), ws.data_ptr(), ws.numel(), cur.cuda_stream))
        else:
            _native.check(self.L.pf_forward(self.handle, ctypes.byref(bt), ws.data_ptr(), ws.numel(), cur.cuda_stream))
        ev = torch.cuda.Event()
        ev.record(cur)
        self.ws_event = ev
        if blob is not None and self.staged_slot is not None and self.dev_blob is not None and blob is self.dev_blob[self.staged_slot]:
            self.blob_free[self.staged_slot] = ev   # stage_images may overwrite this device blob once the forward has read it
        return out

    def param_forward(self, gravity, latitude, with_raw):
        """pf_param_forward on contiguous float32 [n, 2, H, W] / [n, 1, H, W] fields at the working size -> (params [n, 8], raw
        [n, 5] or None), enqueued on the current stream."""
        n = int(gravity.shape[0])
        cur = torch.cuda.current_stream(self.device)
        params = torch.empty((n, 8), dtype=torch.float32, device=self.device)
        raw = torch.empty((n, 5), dtype=torch.float32, device=self.device) if with_raw else None
        ws = self._workspace(_native.check(self.L.pf_param_workspace_bytes(self.handle, n)), cur)
        _native.check(self.L.pf_param_forward(self.handle, n, gravity.data_ptr(), latitude.data_ptr(), params.data_ptr(),
                                              raw.data_ptr() if with_raw else None, ws.data_ptr(), ws.numel(), cur.cuda_stream))
        ev = torch.cuda.Event()
        ev.record(cur)
        self.ws_event = ev
        return params, raw

    def param_train_forward(self, gravity, latitude):
        """pf_param_train_forward on contiguous fields -> raw [n, 5]; the workspace then holds what param_backward reads."""
        n = int(gravity.shape[0])
        cur = torch.cuda.current_stream(self.device)
        raw = torch.empty((n, 5), dtype=torch.float32, device=self.device)
        ws = self._workspace(_native.check(self.L.pf_param_train_workspace_bytes(self.handle, n)), cur)
        _native.check(self.L.pf_param_train_forward(self.handle, n, gravity.data_ptr(), latitude.data_ptr(), raw.data_ptr(), ws.data_ptr(),
                                                    ws.numel(), cur.cuda_stream))
        return raw

    def param_backward(self, n, draw, input_grads):
        """pf_param_backward after param_train_forward(n pairs) -> (gradient buffer, d gravity or None, d latitude or None)."""
        cur = torch.cuda.current_stream(self.device)
        grads = torch.empty(int(self.L.pf_param_grad_numel()), dtype=torch.float32, device=self.device)
        dg = dl = None
        if input_grads:
            dg = torch.empty((n, 2, self.net_h, self.net_w), dtype=torch.float32, device=self.device)
            dl = torch.empty((n, 1, self.net_h, self.net_w), dtype=torch.float32, device=self.device)
        ws = self._workspace(_native.check(self.L.pf_param_train_workspace_bytes(self.handle, n)), cur)
        _native.check(self.L.pf_param_backward(self.handle, n, draw.data_ptr(), grads.data_ptr(), dg.data_ptr() if input_grads else None,
                                               dl.data_ptr() if input_grads else None, ws.data_ptr(), ws.numel(), cur.cuda_stream))
        ev = torch.cuda.Event()
        ev.record(cur)
        self.ws_event = ev
        return grads, dg, dl


class ResizeTransform:
    """The ``aug`` attribute of the reference class (perspectivefields.py:16-67, built at :155).  ``apply_image`` keeps the
    reference's contract -- numpy HWC in, numpy HWC out, uint8 through Pillow's antialiased bilinear resampler (bit-exact
    integer restatement, csrc/prepost.cuh: the same arithmetic ``inference`` uses inside its fused pre-process), any other
    dtype through ``F.interpolate(mode="bilinear", align_corners=False)`` -- but the arithmetic runs on the GPU
    (``pf_op_resize_u8`` / ``pf_op_resize_f32``).  Only the bilinear filter exists here (the one the path uses)."""

    def __init__(self, new_h, new_w, interp=None):
        self.new_h, self.new_w = new_h, new_w
        self.interp = 2 if interp is None else interp          # PIL.Image.BILINEAR == 2

    def apply_image(self, img, interp=None):
        img = np.asarray(img)
        assert len(img.shape) <= 4
        method = self.interp if interp is None else interp
        if method != 2:
            raise NotImplementedError("perspectivefields_b200 implements the BILINEAR resize of the inference path only")
        if not torch.cuda.is_available():
            raise RuntimeError("perspectivefields_b200 has no CPU path: ResizeTransform.apply_image needs a CUDA device")
        L = _native.lib()
        dev = torch.device("cuda", torch.cuda.current_device())
        stream = torch.cuda.current_stream(dev).cuda_stream
        if img.dtype == np.uint8:
            if img.ndim != 3 or img.shape[2] != 3:
                raise TypeError("uint8 images must be (H, W, 3); got %s" % (img.shape,))
            src = torch.from_numpy(np.ascontiguousarray(img)).to(dev)
            out = torch.empty((self.new_h, self.new_w, 3), dtype=torch.uint8, device=dev)
            _native.check(L.pf_op_resize_u8(src.data_ptr(), img.shape[0], img.shape[1], self.new_h, self.new_w, out.data_ptr(), stream))
            return out.cpu().numpy()
        if img.ndim not in (2, 3):
            raise TypeError("float images must be (H, W) or (H, W, C); got %s" % (img.shape,))
        c = 1 if img.ndim == 2 else img.shape[2]
        src = torch.from_numpy(np.ascontiguousarray(img, dtype=np.float32)).to(dev)
        out = torch.empty((self.new_h, self.new_w) + img.shape[2:], dtype=torch.float32, device=dev)
        _native.check(L.pf_op_resize_f32(src.data_ptr(), img.shape[0], img.shape[1], c, self.new_h, self.new_w, out.data_ptr(), stream))
        return out.cpu().numpy().astype(img.dtype, copy=False)


class PerspectiveFields(nn.Module):
    def __init__(self, version="Paramnet-360Cities-edina-centered", logits=True, precision="fp32", resize=None, confidence=False,
                 decode="argmax", tta=None):
        """``logits=False`` (classification variant only, SURVEY.md 8f-3; NOT the reference's behaviour): ``pred_gravity`` /
        ``pred_latitude`` hold the decoded fields ([2,320,320] up-vectors, [1,320,320] degrees) instead of the 73 / 180 raw logits,
        which are then never written (engine option "decode_only"); the ``*_original`` entries are unchanged.

        ``precision``: ``"fp32"`` (default) keeps the reference's fp32 numerics within 1e-3 (three bf16 MMAs per product).
        ``"bf16"`` (opt-in, NOT the reference's numerics) runs every tensor-core product as one bf16 MMA on bf16-rounded operands
        with fp32 accumulation, as ``torch.autocast(dtype=torch.bfloat16)`` would; normalisation, softmax, depthwise convolutions
        and the prediction tails stay fp32.  Outputs then differ from fp32 by about 1e-2 relative (DESIGN.md section 3 lists the
        measured error per output).  It is the engine option "bf16" and survives ``.to()`` / ``load_state_dict``.

        ``resize``: the working size ``(H, W)`` the network runs at, in the reference's ``DATALOADER.RESIZE = [Height, Width]``
        order; ``None`` keeps the yaml's ``[320, 320]``.  H and W must be multiples of 32 in [64, 640] with (H/32) * (W/32) <= 256
        (``ValueError`` otherwise, before any GPU work).  ``cfg.DATALOADER.RESIZE``, ``aug`` and the ``[C, H, W]`` fields
        ``pred_gravity`` / ``pred_latitude`` follow it; ``forward`` expects ``[3, H, W]`` images.  Like ``precision`` it survives
        ``.to()`` / ``load_state_dict``.

        ``confidence=True`` (classification variant only, ``ValueError`` otherwise): every result also carries how sure each head is
        at each pixel, ``max_c softmax(logits)_c`` over all of the head's classes (DESIGN.md section 1, "Head confidence"), in
        [1/NC, 1]: ``pred_gravity_confidence`` / ``pred_latitude_confidence`` [H, W] at the working size and
        ``pred_gravity_confidence_original`` / ``pred_latitude_confidence_original`` [height, width], resampled as the latitude
        map is.  They follow the other keys, whose values are unchanged.  It combines with ``logits``, ``precision`` and
        ``resize`` and survives ``.to()`` / ``load_state_dict``; ``calibrate.fit_camera(..., weights="confidence")`` reads it.

        ``decode``: how the classification heads' logits become fields.  ``"argmax"`` (default) is the reference's decode: the
        argmax bin's centre, so up directions snap to 5-degree and latitudes to 1-degree steps.  ``"subbin"`` (classification
        variant only, ``ValueError`` otherwise; NOT the reference's decode) moves the argmax bin c to c + delta, delta in [-1/2, 1/2]
        the vertex of the parabola through the logits of c and its two neighbours (DESIGN.md section 1, "Sub-bin decode"; engine
        option "subbin").  The fields become continuous and are exact for logits quadratic in the bin distance near the peak; how
        much this helps a trained checkpoint has not been measured.  With ``logits=False``, ``pred_gravity`` / ``pred_latitude``
        hold the refined fields; with ``logits=True`` only the ``_original`` fields change.  Logits, confidence maps and every other
        key are unchanged.  It combines with ``logits``, ``precision``, ``resize`` and ``confidence`` and survives ``.to()`` /
        ``load_state_dict``; ``calibrate.fit_camera`` and ``rectify.level_panoramas`` read the refined fields as they are.

        ``tta``: test-time augmentation.  ``None`` (default) runs each image once.  ``"flip"`` (any variant; NOT the reference's
        behaviour) also runs its left-right mirror, taken before the pre-process, and merges the two heads' outputs at the
        working size (DESIGN.md section 1, "Flip test-time augmentation"; engine option "flip_tta"): up vectors are summed with
        the mirror's x component negated and re-normalised, sin-latitudes averaged, classification logits averaged with the up
        head's classes mirrored.  Decode, confidence, the ``_original`` fields and ParamNet then run on the merged outputs, so
        every key, shape and order is unchanged, and ``pred_gravity`` / ``pred_latitude`` (logits, or the regression fields)
        of a mirrored image are the mirror of the image's bit for bit.  The network runs twice per image; how much this helps a
        trained checkpoint has not been measured.  It combines with ``logits``, ``precision``, ``resize``, ``confidence`` and
        ``decode`` and survives ``.to()`` / ``load_state_dict``.  Any other value is a ``ValueError``."""
        super().__init__()
        zoo = model_zoo[version]  # KeyError for unknown versions, like the reference (perspectivefields.py:127)
        self.version = version
        self.param_on = zoo["param"]
        self._net_hw = check_resize(resize)
        self.cfg = make_cfg(version)
        self.cfg.DATALOADER["RESIZE"] = list(self._net_hw)
        self._variant = VARIANTS[version]
        self.register_buffer("pixel_mean", torch.tensor(PIXEL_MEAN).view(-1, 1, 1), False)
        self.register_buffer("pixel_std", torch.tensor(PIXEL_STD).view(-1, 1, 1), False)
        self.vis_period = self.cfg.VIS_PERIOD
        self.freeze = self.cfg.MODEL.FREEZE
        self.debug_on = self.cfg.DEBUG_ON
        self.input_format = self.cfg.INPUT.FORMAT
        self.aug = ResizeTransform(self._net_hw[0], self._net_hw[1])
        self._schema = dict(checkpoint_schema(version))
        self._ref_state = default_state(version)   # reference-layout weights, host side
        self._engine = None
        self._options = {}
        self._jpeg = None
        if not logits:
            if self._variant["gravity"] != "classification":
                raise ValueError("logits=False only applies to the classification variant (PersNet-360Cities)")
            self._options["decode_only"] = 1
        if not isinstance(confidence, bool):
            raise ValueError(f"confidence must be a bool, got {confidence!r}")
        if confidence and self._variant["gravity"] != "classification":
            raise ValueError(f"confidence=True needs classification heads; {version} regresses its fields (PersNet-360Cities has them)")
        self._confidence = bool(confidence)
        if decode not in ("argmax", "subbin"):
            raise ValueError(f"decode must be 'argmax' or 'subbin', got {decode!r}")
        if decode == "subbin":
            if self._variant["gravity"] != "classification":
                raise ValueError(f"decode='subbin' needs classification heads; {version} regresses its fields (PersNet-360Cities has them)")
            self._options["subbin"] = 1
        if precision not in ("fp32", "bf16"):
            raise ValueError(f"precision must be 'fp32' or 'bf16', got {precision!r}")
        if precision == "bf16":
            self._options["bf16"] = 1
        if not (tta is None or (isinstance(tta, str) and tta == "flip")):
            raise ValueError(f"tta must be None or 'flip', got {tta!r}")
        if tta == "flip":
            self._options["flip_tta"] = 1
        self.training = False
        self._pn_params = None      # param_net_parameters(): trainable ParamNet weights, the source of truth once created
        self._pn_synced = None      # (engine serial, training tensors registered, parameter versions) of the last derivation
        self._init_weights()

    # ------------------------------------------------------------------------------------------ module plumbing
    @property
    def device(self):
        return self.pixel_mean.device

    @staticmethod
    def versions():
        for key in model_zoo:
            print(f"{key}")
            print(f"   - {model_zoo[key]['description']}")

    def train(self, mode=True):
        if mode:
            raise RuntimeError("perspectivefields_b200.PerspectiveFields is inference-only: call .eval()")
        return super().train(False)

    def state_dict(self, *args, destination=None, prefix="", keep_vars=False):
        """The reference's key layout (backbone.*, ll_enc.*, persformer_heads.*, param_net.backbone.*), with
        ``nn.Module.state_dict``'s arguments: entries are added to ``destination`` under ``prefix``; ``keep_vars`` returns the
        stored tensors themselves instead of detached copies."""
        if args:   # legacy positional form: (destination, prefix, keep_vars)
            destination = args[0]
            prefix = args[1] if len(args) > 1 else prefix
            keep_vars = args[2] if len(args) > 2 else keep_vars
        if destination is None:
            import collections
            destination = collections.OrderedDict()
        pn = self._pn_params or {}
        for k, v in self._ref_state.items():
            v = pn.get(k, v)
            destination[prefix + k] = v if keep_vars else v.detach().clone()
        return destination

    def load_state_dict(self, state_dict, strict=True, assign=False):
        missing = [k for k in self._schema if k not in state_dict]
        unexpected = [k for k in state_dict if k not in self._schema]
        errors = []
        for k, v in state_dict.items():
            if k in self._schema:
                if tuple(v.shape) != tuple(self._schema[k]):
                    errors.append(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(self._schema[k])}")
        if strict and (missing or unexpected):
            errors.append(f"missing keys {missing[:5]}..., unexpected keys {unexpected[:5]}...")
        if errors:
            raise RuntimeError("Error(s) in loading state_dict for PerspectiveFields:\n\t" + "\n\t".join(errors))
        for k, v in state_dict.items():
            if k in self._schema:
                self._ref_state[k] = v.detach().to("cpu", self._ref_state[k].dtype).clone()
                if self._pn_params is not None and k in self._pn_params:
                    with torch.no_grad():
                        self._pn_params[k].copy_(v.detach())     # in place: an optimizer holding the parameters keeps working
        self._drop_engine()
        return torch.nn.modules.module._IncompatibleKeys(missing, unexpected)

    def _init_weights(self):
        """perspectivefields.py:178-192."""
        state_dict = load_zoo_checkpoint(model_zoo[self.version]["weights"])
        self.load_state_dict(state_dict, strict=False)  # a no-op on the {"model": ...} wrapper, as in the reference
        if state_dict:
            self.load_state_dict(state_dict["model"], strict=False)

    def _apply(self, fn, *args, **kwargs):
        """``.to()`` / ``.cuda()`` / ``.cpu()``: a move to another device writes the ParamNet parameters back into the host state and
        detaches them from the model (``param_net_parameters()`` then creates a new set on the new device)."""
        old = self.device
        out = super()._apply(fn, *args, **kwargs)
        if getattr(self, "_pn_params", None) is not None and self.device != old:
            for k, p in self._pn_params.items():
                self._ref_state[k] = p.detach().to("cpu", self._ref_state[k].dtype).clone()
            self._pn_params = None
            self._pn_synced = None
        return out

    def _drop_engine(self):
        if self._jpeg is not None and self._engine is not None:
            self._engine.L.pf_jpeg_destroy(self._jpeg)
        self._jpeg = None
        if self._engine is not None:
            self._engine.close()
            self._engine = None

    def _get_engine(self):
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("perspectivefields_b200 has no CPU path: move the model to an H100 with .cuda() first")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if self._engine is None or self._engine.device != dev:
            self._drop_engine()
            with torch.cuda.device(dev):
                eng = _Engine(dev, self.version, self._ref_state, self._net_hw)
            eng.gravity_classes = self._variant["gravity_classes"]
            eng.latitude_classes = self._variant["latitude_classes"]
            for k, v in self._options.items():
                _native.check(eng.L.pf_set_option(eng.handle, k.encode(), v))
            eng.decode_only = bool(self._options.get("decode_only", 0))
            eng.confidence = self._confidence
            self._engine = eng
        self._pn_sync(self._engine)
        return self._engine

    def _pn_sync(self, eng):
        """Re-derives the engine's ParamNet tensors from ``param_net_parameters()`` when a parameter changed (its ``_version``) since
        the last derivation, or the engine is new: ``weights.repack_param_net`` (+ ``param_net_train_weights`` once the backward
        has run) as torch operations on the device, copied in place into the registered tensors (their pointers and the engine's
        cached TMA maps stay valid), enqueued on the current stream."""
        if self._pn_params is None:
            return
        key = (eng.serial, eng.train_ready, tuple(p._version for p in self._pn_params.values()))
        if key == self._pn_synced:
            return
        with torch.no_grad(), torch.cuda.device(eng.device):
            sd = {k: p.detach() for k, p in self._pn_params.items()}
            out = repack_param_net(sd, {})
            if eng.train_ready:
                param_net_train_weights(sd, out)
            for name, t in out.items():
                eng.tensors[name].copy_(t)
        self._pn_synced = key

    # ------------------------------------------------------------------------------------------ ParamNet training
    def param_net_parameters(self):
        """ParamNet's weights as trainable float32 parameters on the model's device: an ordered ``{name: nn.Parameter}`` with every
        ``param_net.backbone.*`` key of the checkpoint (the reference's names and shapes), for any ``torch.optim`` optimizer.
        Created on the first call from the current weights; from then on they are ParamNet's weights: every run that uses
        ParamNet (``inference_batch``, ``forward``, ``param_net``, ``param_losses``, ``param_net_backward``) first re-derives the
        engine's copies if a parameter changed, ``state_dict()`` returns their values and ``load_state_dict`` writes into them in
        place.  They are not registered on the module (``parameters()`` and ``.to()`` behave as before); a move to another device
        writes them back and detaches them.  ``ValueError`` for a variant without ParamNet."""
        if self._variant["param_net"] is None:
            raise ValueError(f"{self.version} has no ParamNet")
        if self._pn_params is None:
            dev = self.device
            self._pn_params = collections.OrderedDict(
                (k, nn.Parameter(self._ref_state[k].detach().to(dev, torch.float32).clone())) for k in self._schema if k.startswith(PN))
            self._pn_synced = None
        return collections.OrderedDict(self._pn_params)

    def param_net_backward(self, predictions, batched_inputs, input_grads=False):
        """``param_losses`` (same inputs, same values bit for bit) plus the gradient of the sum of its losses (detectron2 sums the
        loss dict) with respect to every ``param_net_parameters()`` entry, accumulated into ``.grad`` as ``loss.backward()`` would
        (created if None, else added to).  d loss / d raw head outputs comes from torch autograd through
        ``metrics.param_net_losses``; the ConvNeXt-T backward runs in the engine (pf_param_backward).  With ``input_grads=True`` it
        returns ``(losses, {"pred_gravity": [n, 2, H, W], "pred_latitude": [n, 1, H, W]})``, the gradient with respect to the
        fields (uncentred: the nearest sub-sample's gradient, zero at pixels it does not read).  Does not need train mode and
        nothing synchronises with the host."""
        from . import metrics

        n, g, l = self._param_inputs(predictions)
        v = self._variant
        gt = metrics.param_targets(batched_inputs, n, v["param_net"], v["predict_params"])
        params = self.param_net_parameters()
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            if not eng.train_ready:
                with torch.no_grad():
                    eng.register_train_weights(param_net_train_weights({k: p.detach() for k, p in params.items()}, {}))
                self._pn_sync(eng)
            raw = eng.param_train_forward(g.contiguous(), l.contiguous())
            gt = _batch.upload([gt], torch.float32, raw.device)[0]
            with torch.enable_grad():
                r = raw.detach().requires_grad_(True)
                losses = metrics.param_net_losses(r, gt, v["param_net"], v["predict_params"], float(self.cfg.MODEL.PARAM_DECODER.LOSS_WEIGHT))
                draw, = torch.autograd.grad(sum(losses.values()), r)
            grads, dg, dl = eng.param_backward(n, draw.contiguous(), input_grads)
            with torch.no_grad():
                for name, off, numel in eng.grad_layout():
                    key, t = param_net_grad_to_ref(name, grads[off:off + numel])
                    p = params[key]
                    if p.grad is None:
                        p.grad = t.clone(memory_format=torch.contiguous_format)
                    else:
                        p.grad.add_(t)
        losses = {k: x.detach() for k, x in losses.items()}
        if input_grads:
            return losses, {"pred_gravity": dg, "pred_latitude": dl}
        return losses

    # ------------------------------------------------------------------------------------------ inference API
    @torch.no_grad()
    def inference(self, img_bgr):
        return self.inference_batch([img_bgr])[0]

    @torch.no_grad()
    def inference_batch(self, img_bgr_list):
        """perspectivefields.py:207-221.  uint8 (H, W, 3) images take the fused path (one packed upload, Pillow-exact resize +
        normalise in one kernel); a list containing any other dtype takes the reference's float branch for ALL its members
        (``ResizeTransform.apply_image`` -> non-antialiased ``F.interpolate``, perspectivefields.py:47-66, on the GPU) and then
        the ``forward`` entry.

        CUDA uint8 [H, W, 3] tensors on the model's device (e.g. ``panocam.crop_distortion_views`` crops) take the same fused path
        without leaving the device: one device-to-device pack into a blob, then the same engine call; the results are identical
        to those of the same images passed as numpy arrays.  A list must not mix CUDA tensors with host images (TypeError)."""
        on_dev = [isinstance(im, torch.Tensor) and im.is_cuda for im in img_bgr_list]
        if any(on_dev):
            if not all(on_dev):
                raise TypeError("inference_batch: the list mixes CUDA tensors and host images; pass one kind per call")
            return self._inference_batch_device(img_bgr_list)
        imgs = []
        all_u8 = True
        for im in img_bgr_list:
            im = np.asarray(im)
            if im.ndim != 3 or im.shape[2] != 3:
                raise TypeError("inference expects (H, W, 3) BGR images; got %s %s" % (im.dtype, im.shape))
            if self.input_format == "RGB":
                im = im[:, :, ::-1]
            all_u8 = all_u8 and im.dtype == np.uint8
            imgs.append(np.ascontiguousarray(im))
        if not imgs:
            return []
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            if not all_u8:
                inputs = []
                for im in imgs:
                    r = self.aug.apply_image(im)
                    inputs.append({"image": torch.as_tensor(r.astype("float32").transpose(2, 0, 1)), "height": im.shape[0], "width": im.shape[1]})
                return self.forward(inputs)
            blob, offsets = eng.stage_images(imgs)
            out = eng.forward(len(imgs), [im.shape[0] for im in imgs], [im.shape[1] for im in imgs], blob=blob, offsets=offsets)
        return self._assemble(out)

    def _inference_batch_device(self, imgs):
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("perspectivefields_b200 has no CPU path: move the model to an H100 with .cuda() first")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        for im in imgs:
            if im.dtype != torch.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise TypeError("inference on CUDA tensors expects uint8 (H, W, 3) images; got %s %s" % (im.dtype, tuple(im.shape)))
            if im.device != dev:
                raise ValueError(f"image on {im.device}, the model is on {dev}")
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            if self.input_format == "RGB":
                imgs = [im.flip(2) for im in imgs]
            blob = torch.cat([im.reshape(-1) for im in imgs])      # one device-to-device pack, on the current stream
            offsets = np.zeros(len(imgs), np.int64)
            np.cumsum(np.array([im.numel() for im in imgs[:-1]], np.int64), out=offsets[1:])
            out = eng.forward(len(imgs), [im.shape[0] for im in imgs], [im.shape[1] for im in imgs], blob=blob, offsets=offsets)
        return self._assemble(out)

    # ---- blob-level access for the multi-GPU gather (dist.py): the five output blobs of a batch move as whole buffers ----
    @torch.no_grad()
    def infer_raw(self, img_bgr_list):
        """``inference_batch`` up to (not including) the per-image views: returns the engine's batch outputs
        (``pred_gravity [n,Cg,H,W]`` at the working size, ``pred_latitude``, flat ``gravity_original`` / ``latitude_original`` blobs, ``params [n,8]``)
        plus the host-side offsets / sizes ``assemble_raw`` needs.  uint8 images only."""
        imgs = []
        for im in img_bgr_list:
            im = np.asarray(im)
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3:
                raise TypeError("infer_raw expects (H, W, 3) uint8 BGR images; got %s %s" % (im.dtype, im.shape))
            if self.input_format == "RGB":
                im = im[:, :, ::-1]
            imgs.append(np.ascontiguousarray(im))
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            blob, offsets = eng.stage_images(imgs)
            return eng.forward(len(imgs), [im.shape[0] for im in imgs], [im.shape[1] for im in imgs], blob=blob, offsets=offsets)

    def assemble_raw(self, raw):
        return self._assemble(raw)

    def net_size(self):
        """The working size (H, W): ``cfg.DATALOADER.RESIZE``, the spatial shape of ``pred_gravity`` / ``pred_latitude``."""
        return self._net_hw

    def out_classes(self):
        """Channel counts of ``pred_gravity`` / ``pred_latitude`` as returned (2 / 1 in "decode_only" mode)."""
        if self._options.get("decode_only", 0):
            return (2, 1)
        return (self._variant["gravity_classes"], self._variant["latitude_classes"])

    def decode_batch(self, jpeg_list, max_threads=0):
        """Decode front-end (SURVEY.md 8f-2): a list of JPEG byte strings (what ``cv2.imread`` would read from disk,
        demo/demo.py:151) is decoded on the GPU (nvJPEG, BGR interleaved) into ONE device blob of packed HWC uint8 images -- the
        layout the fused pre-process reads; no host-side pixel buffer exists.  Returns (blob, offsets, heights, widths)."""
        if self.input_format != "BGR":
            raise NotImplementedError("the decode front-end writes BGR (the reference's INPUT.FORMAT)")
        eng = self._get_engine()
        L = eng.L
        with torch.cuda.device(eng.device):
            if self._jpeg is None:
                self._jpeg = ctypes.c_void_p()
                _native.check(L.pf_jpeg_create(eng.device.index, max_threads, ctypes.byref(self._jpeg)))
            n = len(jpeg_list)
            bufs = [np.frombuffer(b, dtype=np.uint8) for b in jpeg_list]
            hs, ws = (ctypes.c_int32 * n)(), (ctypes.c_int32 * n)()
            for i, b in enumerate(bufs):
                h1, w1 = ctypes.c_int32(), ctypes.c_int32()
                _native.check(L.pf_jpeg_info(self._jpeg, b.ctypes.data, b.size, ctypes.byref(h1), ctypes.byref(w1)))
                hs[i], ws[i] = h1.value, w1.value
            sizes = [hs[i] * ws[i] * 3 for i in range(n)]
            offsets = np.zeros(n, np.int64)
            np.cumsum(sizes[:-1], out=offsets[1:])
            offs = (ctypes.c_int64 * n)(*offsets.tolist())
            blob = torch.empty(int(sum(sizes)), dtype=torch.uint8, device=eng.device)
            ptrs = (ctypes.c_void_p * n)(*[b.ctypes.data for b in bufs])
            lens = (ctypes.c_int64 * n)(*[b.size for b in bufs])
            stream = torch.cuda.current_stream(eng.device).cuda_stream
            _native.check(L.pf_jpeg_decode_batch(self._jpeg, n, ptrs, lens, hs, ws, blob.data_ptr(), offs, stream))
        return blob, offsets, list(hs), list(ws)

    @torch.no_grad()
    def inference_batch_encoded(self, jpeg_list, max_threads=0):
        """``inference_batch`` on JPEG byte strings: ``decode_batch`` + the forward on the decoded blob.  Returns the same
        ``list[dict]`` as ``inference_batch`` (up to the decoder: nvJPEG's IDCT / chroma up-sampling round differently from
        libjpeg's, so decoded pixels can differ by a few grey levels from ``cv2.imread``)."""
        if not jpeg_list:
            return []
        blob, offsets, hs, ws = self.decode_batch(jpeg_list, max_threads)
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            out = eng.forward(len(jpeg_list), hs, ws, blob=blob, offsets=offsets)
        return self._assemble(out)

    @torch.no_grad()
    def forward(self, batched_inputs):
        """perspectivefields.py:223-272: ``[{"image": float32 [3,H,W] (resized to the working size, un-normalised), "height", "width"}]``."""
        if any(k in batched_inputs[0] for k in ("gt_gravity", "gt_latitude")) and self.training:
            raise RuntimeError("training is not supported")
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            chw = torch.stack([x["image"].to(eng.device, torch.float32) for x in batched_inputs]).contiguous()
            if tuple(chw.shape[1:]) != (3,) + self._net_hw:
                raise ValueError("forward expects images already resized to [3, %d, %d]" % self._net_hw)
            out = eng.forward(len(batched_inputs), [int(x["height"]) for x in batched_inputs],
                              [int(x["width"]) for x in batched_inputs], chw=chw)
        return self._assemble(out)

    def _assemble(self, out):
        """Result dictionaries: keys and order of persformer_heads.py:83-101 + param_network.py:54-67 / 205-220 +
        perspectivefields.py:261-271."""
        v = self._variant
        n = out["pred_gravity"].shape[0]
        # one unbind / split call per output tensor (not ~12 tensor operations per image: at 256 images per call the per-image
        # Python work was several milliseconds)
        hs, ws = [int(x) for x in out["h"]], [int(x) for x in out["w"]]
        pg, pl = out["pred_gravity"].unbind(0), out["pred_latitude"].unbind(0)
        if len(set(zip(hs, ws))) == 1:
            go_ = out["gravity_original"].view(n, 2, hs[0], ws[0]).unbind(0)
            lo_ = out["latitude_original"].view(n, hs[0], ws[0]).unbind(0)
        else:
            go_ = [t.view(2, h, w) for t, h, w in zip(out["gravity_original"].split([2 * h * w for h, w in zip(hs, ws)]), hs, ws)]
            lo_ = [t.view(h, w) for t, h, w in zip(out["latitude_original"].split([h * w for h, w in zip(hs, ws)]), hs, ws)]
        cols = [c.unbind(0) for c in out["params"].t().unbind(0)] if v["param_net"] else None     # cols[j][i] = params[i, j] (0-dim views)
        zeros = torch.zeros_like(out["params"][:, 0]).unbind(0) if v["param_net"] == "ParamNet" else None
        res = []
        for i in range(n):
            d = {"pred_gravity": pg[i], "pred_gravity_original": go_[i], "pred_latitude": pl[i], "pred_latitude_original": lo_[i],
                 "pred_latitude_original_mode": "deg"}
            if v["param_net"] == "ParamNet":
                d.update({"pred_roll": cols[0][i], "pred_pitch": cols[1][i], "pred_vfov": cols[2][i], "pred_rel_focal": cols[5][i],
                          "pred_general_vfov": cols[2][i], "pred_rel_cx": zeros[i], "pred_rel_cy": zeros[i]})
            elif v["param_net"] == "ParamNetConvNextRegress":
                d.update({"pred_roll": cols[0][i], "pred_pitch": cols[1][i], "pred_general_vfov": cols[2][i], "pred_rel_cx": cols[3][i],
                          "pred_rel_cy": cols[4][i], "pred_rel_focal": cols[5][i]})
            res.append(d)
        if "gravity_confidence" in out:
            hw = [h * w for h, w in zip(hs, ws)]
            for k in ("gravity_confidence", "latitude_confidence", "gravity_confidence_original", "latitude_confidence_original"):
                maps = out[k].unbind(0) if out[k].dim() == 3 else [t.view(h, w) for t, h, w in zip(out[k].split(hw), hs, ws)]
                for i in range(n):
                    res[i]["pred_" + k] = maps[i]
        return res

    # ------------------------------------------------------------------------------------------ scoring API
    def targets_from_fields(self, up, lat, lat_mode="deg"):
        """Ground-truth fields -> the reference's targets dict ``{"gt_gravity", "gt_latitude"}`` (persformer_heads.py:60-70) for
        ``losses``.  ``up``: list of float32 CUDA [H, W, 2] up fields, ``lat``: list of [H, W] latitude maps (``lat_mode`` "deg"
        as ``camera_fields`` / ``crop_equi_views`` return them, or "rad" as ``crop_distortion_views`` does), all at the working
        size.  One launch for the whole list; the rule (this project's, the inverse of the inference decode, DESIGN.md section 1):
        regression gravity ``[n, 2, H, W]`` (the (x, y) components), regression latitude ``sin(lat)`` ``[n, 1, H, W]``;
        classification ``metrics.encode_bin`` / ``metrics.encode_bin_latitude`` labels, int64 ``[n, H, W]``."""
        from . import metrics

        lat_rad = metrics._lat_rad(lat_mode)
        n = len(up)
        if n == 0 or len(lat) != n:
            raise ValueError(f"targets_from_fields needs as many latitude maps as up fields (>= 1), got {len(up)} and {len(lat)}")
        dev = _batch.device(__name__, (), self.device)
        h, w = self._net_hw
        for i in range(n):
            _batch.cuda_f32(up[i], f"up[{i}]", dev)
            _batch.cuda_f32(lat[i], f"lat[{i}]", dev)
            if tuple(up[i].shape) != (h, w, 2) or tuple(lat[i].shape) != (h, w):
                raise ValueError(f"field {i}: up {list(up[i].shape)} / lat {list(lat[i].shape)}; the working size needs [{h}, {w}, 2] / [{h}, {w}]")
        u, la = metrics.batch_view(list(up)), metrics.batch_view(list(lat))
        s = u.stride()
        gc, lc = self._variant["gravity_classes"], self._variant["latitude_classes"]
        gg, gl = metrics.encode_fields((u, s, h, w), (la, la.stride(), h, w), gc, lc, lat_rad)
        return {"gt_gravity": gg, "gt_latitude": gl}

    def losses(self, results, targets):
        """What ``StandardPersformerHeads`` puts into its losses dict (persformer_heads.py:60-70, gravity_head.py:199-235,
        latitude_head.py:221-254) for ``inference_batch`` results and ``targets_from_fields`` targets, over the whole list:
        regression ``gravity-msg-normal-loss``, ``gravity-l2-loss``, ``latitude-msg-normal-loss``, ``latitude-l2-loss``;
        classification ``loss_gravity``, ``loss_latitude``; weights and ignore values from ``cfg``.  Values are 0-dim float32 CUDA
        tensors and nothing synchronises.  Where the reference would stop in ``pdb`` (a mean over no pixel) the value is NaN, as
        it is for a class label outside [0, C) that is not the ignore value.  The ``pred_*`` tensors of one ``inference_batch``
        call are rows of one buffer and are read in place; other lists are stacked once."""
        from . import metrics

        if self._options.get("decode_only", 0):
            raise ValueError("losses needs the logits, which a model built with logits=False does not return")
        n = len(results)
        if n == 0:
            raise ValueError("no results")
        dev = _batch.device(__name__, (), self.device)
        h, w = self._net_hw
        gc, lc = self._variant["gravity_classes"], self._variant["latitude_classes"]
        preds = []
        for key, c in (("pred_gravity", gc), ("pred_latitude", lc)):
            ts = [_batch.cuda_f32(r[key], f"results[{i}][{key!r}]", dev) for i, r in enumerate(results)]
            for i, t in enumerate(ts):
                if tuple(t.shape) != (c, h, w):
                    raise ValueError(f"results[{i}][{key!r}] is {list(t.shape)}, the model's is [{c}, {h}, {w}]")
            p = metrics.batch_view(ts)
            if not p.is_contiguous() or p.data_ptr() % 16:
                p = torch.stack(ts)
            preds.append(p)
        tg = []
        for key, c in (("gt_gravity", gc), ("gt_latitude", lc)):
            t = targets[key]
            reg = c <= 2
            shape, dtype = ((n, c, h, w), torch.float32) if reg else ((n, h, w), torch.int64)
            if not isinstance(t, torch.Tensor) or t.dtype != dtype or tuple(t.shape) != shape or t.device != dev:
                got = f"{t.dtype} {list(t.shape)} on {t.device}" if isinstance(t, torch.Tensor) else type(t).__name__
                raise ValueError(f"targets[{key!r}] must be {dtype} {list(shape)} on {dev}, got {got}")
            tg.append(t.contiguous())
        mc = self.cfg.MODEL
        wg, wl = float(mc.GRAVITY_DECODER.LOSS_WEIGHT), float(mc.LATITUDE_DECODER.LOSS_WEIGHT)
        ig, il = int(mc.GRAVITY_DECODER.IGNORE_VALUE), int(mc.LATITUDE_DECODER.IGNORE_VALUE)
        L = _native.lib()
        with torch.cuda.device(dev):
            ws = _batch.workspace(L.pf_head_losses_workspace(n, h, w, gc, lc), dev)
            keys = (("gravity-msg-normal-loss", "gravity-l2-loss", "latitude-msg-normal-loss", "latitude-l2-loss") if gc == 2
                    else ("loss_gravity", "loss_latitude"))
            out = torch.empty(len(keys), dtype=torch.float32, device=dev)
            stream = torch.cuda.current_stream(dev).cuda_stream
            _native.check(L.pf_head_losses(dev.index, n, h, w, gc, preds[0].data_ptr(), tg[0].data_ptr(), lc, preds[1].data_ptr(),
                                           tg[1].data_ptr(), ig, il, wg, wl, out.data_ptr(), ws.data_ptr(), ws.numel(), stream))
        return dict(zip(keys, out.unbind(0)))

    # ------------------------------------------------------------------------------------------ ParamNet on given fields
    def _param_inputs(self, predictions):
        """Checks of ``param_net`` / ``param_losses`` (all before any GPU work) -> (n, pred_gravity, pred_latitude)."""
        if self._variant["param_net"] is None:
            raise ValueError(f"{self.version} has no ParamNet")
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("perspectivefields_b200 has no CPU path: move the model to an H100 with .cuda() first")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        h, w = self._net_hw
        ts = []
        for key, c in (("pred_gravity", 2), ("pred_latitude", 1)):
            if key not in predictions:
                raise KeyError(f"predictions has no {key!r}")
            t = _batch.cuda_f32(predictions[key], f"predictions[{key!r}]", dev)
            if t.dim() != 4 or tuple(t.shape[1:]) != (c, h, w):
                raise ValueError(f"predictions[{key!r}] is {list(t.shape)}, the working size needs [n, {c}, {h}, {w}]")
            ts.append(t)
        n = int(ts[0].shape[0])
        if n == 0:
            raise ValueError("predictions hold no fields (n = 0)")
        if int(ts[1].shape[0]) != n:
            raise ValueError(f"{n} gravity fields but {int(ts[1].shape[0])} latitude fields")
        return n, ts[0], ts[1]

    def _param_run(self, gravity, latitude, with_raw):
        eng = self._get_engine()
        with torch.cuda.device(eng.device):
            return eng.param_forward(gravity.contiguous(), latitude.contiguous(), with_raw)

    @torch.no_grad()
    def param_net(self, predictions, batched_inputs=None):
        """The reference's ``param_net(predictions)`` in eval mode (param_network.py:46-69 ``ParamNet``, :193-221
        ``ParamNetConvNextRegress``) on any fields: ``predictions["pred_gravity"]`` float32 [n, 2, H, W] up vectors and
        ``["pred_latitude"]`` [n, 1, H, W] sin(latitude) on the model's device at the working size (what the regression heads
        return, or the ``gt_gravity`` / ``gt_latitude`` of ``targets_from_fields``).  The fields are used as given (no
        renormalisation or clamp; NaN propagates); the run is the ParamNet section of the forward, so the forward's own fields
        give its parameters bit for bit.  Returns the keys of the variant's class, in its order: ``pred_roll, pred_pitch,
        pred_vfov, pred_rel_focal`` (centred) or ``pred_roll, pred_pitch, pred_general_vfov, pred_rel_cx, pred_rel_cy,
        pred_rel_focal`` (uncentred), each a float32 [n] view of one device tensor (``pred_rel_focal`` too, unlike the
        reference's host tensor of the uncentred class).  ``batched_inputs`` is ignored, as in the reference's eval branch."""
        n, g, l = self._param_inputs(predictions)
        params, _ = self._param_run(g, l, False)
        if self._variant["param_net"] == "ParamNet":
            cols = (("pred_roll", 0), ("pred_pitch", 1), ("pred_vfov", 2), ("pred_rel_focal", 5))
        else:
            cols = (("pred_roll", 0), ("pred_pitch", 1), ("pred_general_vfov", 2), ("pred_rel_cx", 3), ("pred_rel_cy", 4), ("pred_rel_focal", 5))
        return {k: params[:, j] for k, j in cols}

    @torch.no_grad()
    def param_losses(self, predictions, batched_inputs):
        """The losses of the reference's ``param_net(predictions, batched_inputs)`` in training mode (param_network.py:71-128,
        :223-241) for fields as ``param_net`` takes them and targets ``batched_inputs[i]`` holding host numbers in degrees:
        ``roll``, ``pitch``, ``vfov`` (centred; ``{"param-l1-loss"}``) or the keys of ``cfg.MODEL.PARAM_DECODER.PREDICT_PARAMS``
        (uncentred; ``{"param/<key>-loss"}`` per key), weighted by ``cfg.MODEL.PARAM_DECODER.LOSS_WEIGHT``
        (``metrics.param_net_losses`` states the rule).  Values are 0-dim float32 device tensors and nothing synchronises."""
        from . import metrics

        n, g, l = self._param_inputs(predictions)
        v = self._variant
        gt = metrics.param_targets(batched_inputs, n, v["param_net"], v["predict_params"])
        _, raw = self._param_run(g, l, True)
        with torch.cuda.device(raw.device):
            gt = _batch.upload([gt], torch.float32, raw.device)[0]
        return metrics.param_net_losses(raw, gt, v["param_net"], v["predict_params"], float(self.cfg.MODEL.PARAM_DECODER.LOSS_WEIGHT))

    def set_option(self, name, value):
        """Engine options (see pf_set_option in include/pf_b200.h), e.g. ``set_option("pdl", 0)``."""
        eng = self._get_engine()
        _native.check(eng.L.pf_set_option(eng.handle, name.encode(), int(value)))
        self._options[name] = int(value)
        eng.decode_only = bool(self._options.get("decode_only", 0))

    # ------------------------------------------------------------------------------------------ test hooks
    def debug_taps(self, enable=True):
        eng = self._get_engine()
        _native.check(eng.L.pf_debug_enable(eng.handle, 1 if enable else 0))
        eng.workspace = None

    def read_taps(self):
        eng = self._get_engine()
        L, out = eng.L, {}
        stream = torch.cuda.current_stream(eng.device).cuda_stream
        for i in range(L.pf_debug_count(eng.handle)):
            name = L.pf_debug_name(eng.handle, i)
            numel = L.pf_debug_numel(eng.handle, name)
            t = torch.empty(numel, dtype=torch.float32, device=eng.device)
            _native.check(L.pf_debug_copy(eng.handle, name, t.data_ptr(), numel, stream))
            out[name.decode()] = t
        torch.cuda.synchronize(eng.device)
        return out
