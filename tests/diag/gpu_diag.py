"""First-contact diagnostics on the GPU box: every operator against torch, then the whole forward against the oracle,
tap by tap.  Writes a plain-text report to diag_out/diag.txt (also printed).  Test infrastructure, not product."""
import ctypes
import os
import sys
import time
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
import torch.nn.functional as F

import pf_test_util as U
from perspectivefields_b200 import _native

torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
LINES = []


def say(*a):
    s = " ".join(str(x) for x in a)
    print(s, flush=True)
    LINES.append(s)


def guarded(name, fn):
    try:
        fn()
    except Exception:
        say(f"[{name}] EXCEPTION\n" + traceback.format_exc())


def ops():
    L = _native.lib()
    g = torch.Generator(device="cpu").manual_seed(1)
    rn = lambda *s: torch.randn(*s, generator=g)
    cases = [  # B,H,W,Cin,N,K,stride,pad,in_relu,act,res,res_relu
        (2, 20, 20, 64, 256, 3, 1, 1, 0, 0, 0, 0), (2, 20, 20, 256, 256, 3, 1, 1, 1, 1, 0, 0), (1, 23, 17, 256, 256, 3, 1, 1, 0, 0, 1, 1),
        (1, 1, 700, 320, 640, 1, 1, 0, 0, 0, 0, 0), (1, 1, 300, 96, 384, 1, 1, 0, 0, 2, 0, 0), (1, 1, 130, 384, 96, 1, 1, 0, 0, 0, 1, 0),
        (2, 80, 80, 64, 64, 8, 8, 0, 0, 0, 0, 0), (2, 40, 40, 64, 128, 3, 2, 1, 0, 0, 0, 0), (1, 24, 24, 64, 32, 3, 1, 1, 0, 1, 0, 0),
        (1, 16, 16, 96, 192, 2, 2, 0, 0, 0, 0, 0), (1, 40, 40, 320, 64, 3, 1, 1, 0, 1, 0, 0)]
    for (B, H, W, Cin, N, K, s, p, ir, act, res, rr) in cases:
        x = rn(B, Cin, H, W).cuda()
        w = rn(N, Cin, K, K) / (Cin * K * K) ** 0.5
        b = rn(N)
        xin = F.relu(x) if ir else x
        ref = F.conv2d(xin.double(), w.double().cuda(), b.double().cuda(), stride=s, padding=p)
        if act == 1: ref = F.relu(ref)
        if act == 2: ref = F.gelu(ref)
        r = None
        if res:
            r = rn(*ref.shape).cuda()
            ref = ref + (F.relu(r) if rr else r).double()
            r = r.permute(0, 2, 3, 1).contiguous()
        y = U.conv_gemm(x.permute(0, 2, 3, 1).contiguous(), w, b, s, p, ir, act, r, rr)
        say(f"conv_gemm B{B} {H}x{W} Cin{Cin} N{N} k{K} s{s} p{p} relu_in{ir} act{act} res{res}/{rr}: rel {U.rel_err(y.permute(0, 3, 1, 2), ref):.3g}")
    # layernorm
    for C in (64, 96, 128, 320, 512, 768):
        x = rn(777, C).cuda() * 3 + 1; w = rn(C).cuda(); b = rn(C).cuda(); y = torch.empty_like(x)
        _native.check(L.pf_op_layernorm(x.data_ptr(), y.data_ptr(), 777, C, w.data_ptr(), b.data_ptr(), 1e-6, U.stream_ptr()))
        say(f"layernorm C{C}: rel {U.rel_err(y, F.layer_norm(x.double(), (C,), w.double(), b.double(), 1e-6)):.3g}")
    # attention
    for (B, N, heads) in ((2, 6400, 1), (2, 1600, 2), (1, 400, 5), (1, 100, 8), (1, 77, 2)):
        C = heads * 64
        q = rn(B, N, C).cuda(); kv = rn(B, 100, 2 * C).cuda(); o = torch.empty_like(q)
        _native.check(L.pf_op_attention_tc(q.data_ptr(), kv.data_ptr(), o.data_ptr(), B, N, C, heads, U.stream_ptr()))
        qh = q.double().reshape(B, N, heads, 64).permute(0, 2, 1, 3)
        kvh = kv.double().reshape(B, 100, 2, heads, 64).permute(2, 0, 3, 1, 4)
        ref = ((qh @ kvh[0].transpose(-2, -1)) * 0.125).softmax(-1) @ kvh[1]
        say(f"attention B{B} N{N} heads{heads}: rel {U.rel_err(o, ref.transpose(1, 2).reshape(B, N, C)):.3g}")
    # depthwise convs, upsample
    x = rn(2, 256, 20, 20).cuda(); w = rn(256, 1, 3, 3).cuda(); b = rn(256).cuda()
    xh = x.permute(0, 2, 3, 1).contiguous(); y = torch.empty_like(xh)
    _native.check(L.pf_op_dwconv3x3_gelu(xh.data_ptr(), y.data_ptr(), 2, 20, 20, 256, w.reshape(256, 9).t().contiguous().data_ptr(), b.data_ptr(), U.stream_ptr()))
    say(f"dwconv3x3_gelu: rel {U.rel_err(y.permute(0, 3, 1, 2), F.gelu(F.conv2d(x.double(), w.double(), b.double(), padding=1, groups=256))):.3g}")
    x = rn(2, 96, 16, 16).cuda(); w = rn(96, 1, 7, 7).cuda(); b = rn(96).cuda()
    xh = x.permute(0, 2, 3, 1).contiguous(); y = torch.empty_like(xh)
    _native.check(L.pf_op_dwconv7x7(xh.data_ptr(), y.data_ptr(), 2, 16, 16, 96, w.reshape(96, 49).t().contiguous().data_ptr(), b.data_ptr(), U.stream_ptr()))
    say(f"dwconv7x7: rel {U.rel_err(y.permute(0, 3, 1, 2), F.conv2d(x.double(), w.double(), b.double(), padding=3, groups=96)):.3g}")
    x = rn(2, 64, 10, 13).cuda(); xh = x.permute(0, 2, 3, 1).contiguous(); y = torch.empty(2, 20, 26, 64, device="cuda")
    _native.check(L.pf_op_upsample2x(xh.data_ptr(), y.data_ptr(), 2, 10, 13, 64, U.stream_ptr()))
    say(f"upsample2x: rel {U.rel_err(y.permute(0, 3, 1, 2), F.interpolate(x, scale_factor=2, mode='bilinear', align_corners=False)):.3g}")
    # preprocess vs Pillow (must be exact)
    from PIL import Image
    for (h, w) in ((480, 640), (240, 320), (320, 320), (721, 900), (1536, 2048), (33, 47), (512, 512)):
        img = np.random.RandomState(h + w).randint(0, 256, (h, w, 3), dtype=np.uint8)
        ref = np.asarray(Image.fromarray(img).resize((320, 320), Image.BILINEAR)).astype(np.float32) - np.array([103.53, 116.28, 123.675], np.float32)
        d = torch.from_numpy(img).cuda(); y = torch.empty(320, 320, 4, device="cuda")
        mean = (ctypes.c_float * 3)(103.53, 116.28, 123.675); std = (ctypes.c_float * 3)(1, 1, 1)
        _native.check(L.pf_op_preprocess(d.data_ptr(), h, w, mean, std, y.data_ptr(), U.stream_ptr()))
        torch.cuda.synchronize()
        diff = (y[..., :3].cpu().numpy() - ref)
        say(f"preprocess {h}x{w}: max abs diff {np.abs(diff).max():.3g} (exact expected), mismatches {(diff != 0).sum()}")


def full(version, n_img=2):
    from oracle import model as om, weights_gen as wg
    t = time.time()
    m, sd = U.make_model(version)
    imgs = (wg.synth_images(1, 480, 640, 0) + wg.smooth_images(1, 360, 500, 0))[:n_img]
    m.debug_taps(True)
    out = m.inference_batch(imgs)
    torch.cuda.synchronize()
    taps = m.read_taps()
    say(f"[{version}] product forward ok in {time.time() - t:.1f}s, {len(taps)} taps, launches so far {_native.lib().pf_kernel_launch_count()}")
    otaps = {}
    ora = om.inference_batch(sd, version, imgs, otaps)
    B = len(imgs)

    def nchw_tokens(t):  # oracle [B, N, C] tokens or [B,C,H,W] -> NHWC flat
        return t if t.dim() == 3 else t.permute(0, 2, 3, 1)

    for name, t in taps.items():
        ref = None
        if name == "pre":
            ref = torch.stack([om.preprocess(im) for im in imgs]) - torch.tensor([103.53, 116.28, 123.675]).view(1, 3, 1, 1)
            ref = F.pad(ref.permute(0, 2, 3, 1), (0, 1))
        elif name == "ll":
            ref = otaps["ll"].permute(0, 2, 3, 1)
        elif name.startswith("mit."):
            ref = otaps.get(name)
        elif name.startswith("head.proc") or name.startswith("head.fusion") or name in ("head.conv0", "head.conv1"):
            k = name[5:]
            ref = torch.cat([otaps["g." + k], otaps["l." + k]], 1).permute(0, 2, 3, 1)
        elif name.startswith("cnx.s"):
            ref = otaps[name].permute(0, 2, 3, 1)
        if ref is None:
            say(f"  tap {name}: (no oracle counterpart)")
            continue
        ref = ref.contiguous().reshape(-1)
        if ref.numel() != t.numel():
            say(f"  tap {name}: SIZE MISMATCH product {t.numel()} oracle {ref.numel()}")
            continue
        say(f"  tap {name:22s} rel {U.rel_err(t, ref):.3g}")
    for i in range(B):
        for k, v in ora[i].items():
            if isinstance(v, str):
                continue
            say(f"  out[{i}] {k:24s} {tuple(v.shape)} rel {U.rel_err(out[i][k], v):.3g}")
    m.debug_taps(False)
    # quick timing, batch 8
    imgs8 = wg.synth_images(8, 480, 640, 1)
    for _ in range(2):
        m.inference_batch(imgs8)
    torch.cuda.synchronize()
    t = time.time()
    for _ in range(3):
        m.inference_batch(imgs8)
    torch.cuda.synchronize()
    say(f"[{version}] batch 8: {(time.time() - t) / 3 * 1000:.1f} ms/batch -> {8 * 3 / (time.time() - t):.1f} img/s (wall, incl. H2D)")


if __name__ == "__main__":
    os.makedirs(os.path.join(ROOT, "diag_out"), exist_ok=True)
    say(torch.cuda.get_device_name(0), torch.__version__)
    guarded("ops", ops)
    for ver in sys.argv[1:] or ["Paramnet-360Cities-edina-centered"]:
        guarded(ver, lambda: full(ver))
    with open(os.path.join(ROOT, "diag_out", "diag.txt"), "w") as f:
        f.write("\n".join(LINES) + "\n")
