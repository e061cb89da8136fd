"""Multi-GPU ``inference_batch`` (SURVEY.md section 8e): one process per GPU (``torch.distributed`` for the rendezvous; NCCL over
NVLink on a multi-GPU box, gloo in the CPU tests).  The path has no cross-image dependency, so the list is sharded in contiguous
chunks, every rank runs the ordinary single-GPU path on its shard in micro-batches, and the results are gathered to ONE rank so
that the caller gets the ``list[dict]`` a single-GPU call would return -- bit-identical per image, tensors on that rank's device
(where the reference would have put them).

The gather moves each micro-batch's five output blobs (not per-image tensors) with grouped point-to-point transfers on a side
stream, so the transfer of micro-batch k overlaps the forward of micro-batch k+1:

* ``PfCommTransport``: ``pf_gather`` of libpf_b200.so -- grouped ``ncclSend`` / ``ncclRecv`` issued from C on the side stream
  (include/pf_b200.h); the communicator's unique id travels through ``torch.distributed`` (plumbing).
* ``TorchTransport``: ``torch.distributed.batch_isend_irecv`` (gloo on CPU in the tests; also works with the NCCL backend).
"""
import ctypes
import os
import time

import numpy as np
import torch
import torch.distributed as dist

_NET = 320          # default working size (DATALOADER.RESIZE); a model built with ``resize`` passes its own net_hw
_BLOBS = ("pred_gravity", "pred_latitude", "gravity_original", "latitude_original", "params")


def shard_bounds(n, world):
    """Contiguous shards of ceil(n / world) images: [(lo, hi)] per rank (empty shards at the tail are legal)."""
    per = -(-n // world) if n else 0
    return [(min(r * per, n), min((r + 1) * per, n)) for r in range(world)]


def micro_batches(lo, hi, mb):
    """[(a, b)] covering [lo, hi) in steps of mb images."""
    return [(a, min(a + mb, hi)) for a in range(lo, hi, mb)] if hi > lo else []


def _result_spec(variant, h, w, net_hw=(_NET, _NET)):
    """(key, shape) of every tensor in one image's result dict, in order (SURVEY.md section 8a)."""
    g, l = variant["gravity_classes"], variant["latitude_classes"]
    nh, nw = net_hw
    spec = [("pred_gravity", (g, nh, nw)), ("pred_gravity_original", (2, h, w)), ("pred_latitude", (l, nh, nw)),
            ("pred_latitude_original", (h, w))]
    if variant["param_net"] == "ParamNet":
        spec += [(k, ()) for k in ("pred_roll", "pred_pitch", "pred_vfov", "pred_rel_focal", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy")]
    elif variant["param_net"] == "ParamNetConvNextRegress":
        spec += [(k, ()) for k in ("pred_roll", "pred_pitch", "pred_general_vfov", "pred_rel_cx", "pred_rel_cy", "pred_rel_focal")]
    return spec


def blob_numels(out_classes, sizes, net_hw=(_NET, _NET)):
    """Element counts of the five output blobs of a micro-batch whose images have the given (h, w) sizes, for a model whose
    working size is ``net_hw`` (``PerspectiveFields.net_size()``)."""
    g, l = out_classes
    m = len(sizes)
    hw = sum(h * w for h, w in sizes)
    nhw = net_hw[0] * net_hw[1]
    return {"pred_gravity": m * g * nhw, "pred_latitude": m * l * nhw, "gravity_original": 2 * hw, "latitude_original": hw,
            "params": m * 8}


def empty_raw(out_classes, sizes, device, net_hw=(_NET, _NET)):
    """Receive buffers with the layout ``PerspectiveFields.infer_raw`` produces for these image sizes."""
    g, l = out_classes
    nh, nw = net_hw
    m = len(sizes)
    h = np.asarray([s[0] for s in sizes], np.int32)
    w = np.asarray([s[1] for s in sizes], np.int32)
    hw = h.astype(np.int64) * w.astype(np.int64)
    g_off, l_off = np.zeros(m, np.int64), np.zeros(m, np.int64)
    np.cumsum(2 * hw[:-1], out=g_off[1:])
    np.cumsum(hw[:-1], out=l_off[1:])
    return {"pred_gravity": torch.empty((m, g, nh, nw), dtype=torch.float32, device=device),
            "pred_latitude": torch.empty((m, l, nh, nw), dtype=torch.float32, device=device),
            "gravity_original": torch.empty(int(2 * hw.sum()), dtype=torch.float32, device=device),
            "latitude_original": torch.empty(int(hw.sum()), dtype=torch.float32, device=device),
            "params": torch.empty((m, 8), dtype=torch.float32, device=device),
            "g_off": g_off, "l_off": l_off, "h": h, "w": w}


class TorchTransport:
    """Grouped point-to-point transfers through ``torch.distributed`` (gloo / NCCL backend of the default group)."""

    def __init__(self, group=None):
        self.group = group
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)

    def exchange(self, root, tensors, peers, stream=None):
        """Non-root: send ``tensors`` to root.  Root: receive tensors[i] from rank peers[i]."""
        ops = []
        for i, t in enumerate(tensors):
            if self.rank == root:
                ops.append(dist.P2POp(dist.irecv, t, peers[i], self.group))
            else:
                ops.append(dist.P2POp(dist.isend, t, root, self.group))
        if ops:
            for req in dist.batch_isend_irecv(ops):
                req.wait()

    def close(self):
        pass


class PfCommTransport:
    """``pf_comm_*`` / ``pf_gather`` of libpf_b200.so: one NCCL communicator owned by the library, grouped ncclSend / ncclRecv
    enqueued on the given CUDA stream from C."""

    def __init__(self, device, group=None):
        from . import _native

        self.N = _native
        self.L = _native.lib()
        self.rank, self.world = dist.get_rank(group), dist.get_world_size(group)
        self.device = torch.device(device)
        uid = (ctypes.c_uint8 * 128)()
        if self.rank == 0:
            _native.check(self.L.pf_comm_unique_id(uid))
        box = [bytes(uid)]
        dist.broadcast_object_list(box, src=0, group=group)     # plumbing: 128 bytes
        uid = (ctypes.c_uint8 * 128).from_buffer_copy(box[0])
        self.handle = ctypes.c_void_p()
        with torch.cuda.device(self.device):
            _native.check(self.L.pf_comm_create(self.device.index, self.rank, self.world, uid, ctypes.byref(self.handle)))
        self.bytes_moved = 0

    def exchange(self, root, tensors, peers, stream=None):
        n = len(tensors)
        if n == 0:
            return
        st = stream if stream is not None else torch.cuda.current_stream(self.device)
        ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tensors])
        nbytes = (ctypes.c_int64 * n)(*[t.numel() * t.element_size() for t in tensors])
        pr = (ctypes.c_int32 * n)(*[int(p) for p in peers]) if self.rank == root else None
        self.N.check(self.L.pf_gather(self.handle, root, n, ptrs, nbytes, pr, st.cuda_stream))
        self.bytes_moved += sum(nbytes)

    def close(self):
        if self.handle:
            self.L.pf_comm_destroy(self.handle)
            self.handle = ctypes.c_void_p()


def _sizes(imgs):
    return [(int(im.shape[0]), int(im.shape[1])) for im in imgs]


def inference_batch_sharded(model, img_bgr_list, gather_to=0, group=None, micro_batch=32, transport=None, wait=True):
    """Every rank passes the SAME list; rank r runs the model on its shard, ``micro_batch`` images at a time.  With ``gather_to``
    = a rank, that rank returns the full ``list[dict]`` in input order (tensors on its device) and the other ranks return their
    own shard's results; with ``gather_to=None`` nothing is exchanged.  ``transport``: a ``PfCommTransport`` / ``TorchTransport``
    to reuse across calls (default: a ``TorchTransport`` on ``group``).

    ``wait=False`` (pipelined calls): the caller's stream is NOT made to wait for the transfers; the function returns
    ``(results, event)`` and the caller waits on ``event`` (recorded on the side stream) before touching gathered tensors -- the
    gather of call k then overlaps the forward of call k+1.

    The receives of a round are posted only after the gathering rank's OWN forward of that round has finished: an NCCL receive
    kernel posted earlier would sit on its SMs spinning for the peers' data while the forward's persistent kernels (one
    225 KB-shared-memory CTA per SM) need every SM.

    ``model`` provides ``infer_raw(imgs) -> raw`` (the five output blobs of one micro-batch + host metadata),
    ``assemble_raw(raw) -> list[dict]`` and ``out_classes()`` (``PerspectiveFields`` does), optionally ``net_size()`` (the working
    size of ``pred_gravity`` / ``pred_latitude``; 320 x 320 when absent).  A model built with ``confidence=True`` is refused
    (``ValueError``): the gather does not carry the confidence maps."""
    if getattr(model, "_confidence", False):
        raise ValueError("inference_batch_sharded does not gather the confidence maps of a confidence=True model; "
                         "call inference_batch on each rank instead")
    if not dist.is_available() or not dist.is_initialized():
        return model.inference_batch(img_bgr_list)
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    n = len(img_bgr_list)
    bounds = shard_bounds(n, world)
    lo, hi = bounds[rank]
    if gather_to is None or world == 1:
        return [d for a, b in micro_batches(lo, hi, micro_batch) for d in model.inference_batch(img_bgr_list[a:b])]
    tr = transport if transport is not None else TorchTransport(group)
    device = torch.device(model.device)
    on_gpu = device.type == "cuda"
    cur = torch.cuda.current_stream(device) if on_gpu else None
    side = _side_stream(model, device) if on_gpu else None
    if on_gpu:
        side.wait_stream(cur)
    sizes = _sizes(img_bgr_list)
    classes = model.out_classes()
    net_hw = tuple(model.net_size()) if hasattr(model, "net_size") else (_NET, _NET)   # the blobs follow the model's working size
    my_mbs = micro_batches(lo, hi, micro_batch)
    rounds = max(len(micro_batches(a, b, micro_batch)) for a, b in bounds)
    results = [None] * n
    keep = []
    trace = {} if os.environ.get("PF_DIST_TRACE") else None
    t_ = time.perf_counter()

    def lap(name):
        nonlocal t_
        if trace is not None:
            now = time.perf_counter()
            trace[name] = trace.get(name, 0.0) + (now - t_) * 1000
            t_ = now
    for k in range(rounds):
        raw = None
        if k < len(my_mbs):
            a, b = my_mbs[k]
            raw = model.infer_raw(img_bgr_list[a:b])
            lap("infer_raw")
            for i, d in zip(range(a, b), model.assemble_raw(raw)):
                results[i] = d
            lap("assemble_own")
        # exchange of round k on the side stream, after this rank's forward of round k; the next round's forward (enqueued on
        # the compute stream by the next loop iteration) overlaps it
        done = None
        if on_gpu:
            done = torch.cuda.Event()
            done.record(cur)
        if rank == gather_to:
            bufs, peers, metas = [], [], []
            ctx = torch.cuda.stream(side) if on_gpu else _Null()
            if on_gpu:
                side.wait_event(done)            # (see the docstring: no receive kernel while this rank's forward runs)
            with ctx:
                for r, (ra, rb) in enumerate(bounds):
                    mbs = micro_batches(ra, rb, micro_batch)
                    if r == rank or k >= len(mbs):
                        continue
                    a, b = mbs[k]
                    recv = empty_raw(classes, sizes[a:b], device, net_hw)
                    for key in _BLOBS:
                        bufs.append(recv[key])
                        peers.append(r)
                    metas.append((a, b, recv))
                lap("alloc_recv")
                tr.exchange(gather_to, bufs, peers, side)
                lap("exchange_call")
            for a, b, recv in metas:
                for i, d in zip(range(a, b), model.assemble_raw(recv)):
                    results[i] = d
                if on_gpu:
                    for key in _BLOBS:
                        recv[key].record_stream(cur)     # allocated on the side stream, consumed by the caller on `cur`
            lap("assemble_remote")
        elif raw is not None:
            if on_gpu:
                side.wait_event(done)
            tr.exchange(gather_to, [raw[key] for key in _BLOBS], None, side)
            lap("exchange_call")
            keep.append(raw)
            if on_gpu:
                for key in _BLOBS:
                    raw[key].record_stream(side)
    ev = None
    if on_gpu:
        if wait:
            cur.wait_stream(side)    # the caller's stream sees complete results
        else:
            ev = torch.cuda.Event()
            ev.record(side)
    if trace is not None:
        print(f"[pf dist rank {rank}] host ms: " + ", ".join(f"{k} {v:.2f}" for k, v in trace.items()), flush=True)
    out = results if rank == gather_to else [results[i] for i in range(lo, hi)]
    return out if wait else (out, ev)


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def _side_stream(model, device):
    s = getattr(model, "_pf_comm_stream", None)
    if s is None or s.device != device:
        s = torch.cuda.Stream(device=device)
        try:
            model._pf_comm_stream = s
        except Exception:
            pass
    return s
