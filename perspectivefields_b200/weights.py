"""Checkpoint -> kernel-layout repack (host side, once per load_state_dict).

Input: the reference's ``{"model": state_dict}`` layout (perspective2d/perspectivefields.py:178-192; key schema in
SURVEY.md appendix A).  Output: ``{name: tensor}`` with the names ``csrc/pf_b200.cu:resolve_weights`` looks up.

* GEMM layers (every nn.Linear / groups=1 nn.Conv2d except the ParamNet stem): ``<n>.whi`` / ``<n>.wlo`` = bf16
  hi / lo planes of the [N][K] weight, K ordered (ky, kx, ci); ``<n>.b`` fp32 bias.
* Decoder-head ``linear_c{l}`` (1x1, C->768) followed by ``linear_c{l}_proc`` (3x3, 768->256) has no non-linearity in
  between (gravity_head.py:146-149): composed exactly, in fp64, into one 3x3 conv C->256.  The Linear's bias goes
  through the zero-padded 3x3 conv, so its contribution depends on which taps fall inside the image: 9 bias vectors,
  one per border class (top/mid/bottom x left/mid/right).  Both heads share the input, so their composed weights are
  concatenated along N (512 outputs).
* The two heads' RefineNet convs are stored as two weight groups of one grouped launch.
* Eval-mode BatchNorm of ``ll_enc`` is folded into its conv (perspectivefields.py:73-83).
* The ParamNet stem, depthwise and prediction layers stay fp32 in the layouts the CUDA-core kernels read.
"""
import torch

from .variants import CNX_DEPTHS, CNX_DIMS, MIT_DEPTHS, MIT_DIMS, MIT_SR


def split_hi_lo(w):
    """fp64/fp32 tensor -> (bf16 hi, bf16 lo) with hi + lo ~= w to 16 significant bits."""
    w = w.double()
    hi = w.to(torch.bfloat16)
    lo = (w - hi.double()).to(torch.bfloat16)
    return hi.contiguous(), lo.contiguous()


def _conv_to_nk(w):
    """[Cout, Cin, kh, kw] -> [Cout, kh*kw*Cin] with k = (ky, kx, ci)."""
    return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1)


def _put_gemm(out, name, w_nk, bias):
    hi, lo = split_hi_lo(w_nk)
    out[name + ".whi"], out[name + ".wlo"] = hi, lo
    out[name + ".b"] = bias.float().contiguous()


def _put_ln(out, name, sd, key):
    out[name + ".w"] = sd[key + ".weight"].float().contiguous()
    out[name + ".b"] = sd[key + ".bias"].float().contiguous()


def _stem(w):
    """[Cout, 3, kh, kw] -> [(ky, kx, ci)][Cout] fp32."""
    return w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]).float().contiguous()


def _compose_proc(sd, head, lvl):
    p = f"persformer_heads.{head}."
    W1 = sd[f"{p}linear_c{lvl}.proj.weight"].double()      # [768, C]
    b1 = sd[f"{p}linear_c{lvl}.proj.bias"].double()        # [768]
    W3 = sd[f"{p}linear_c{lvl}_proc.weight"].double()      # [256, 768, 3, 3]
    b3 = sd[f"{p}linear_c{lvl}_proc.bias"].double()        # [256]
    Wc = torch.einsum("oeyx,ec->ocyx", W3, W1)             # [256, C, 3, 3]
    btap = torch.einsum("oeyx,e->yxo", W3, b1)             # [3, 3, 256]
    valid = {0: (1, 2), 1: (0, 1, 2), 2: (0, 1)}           # border class -> taps that fall inside the image
    bias = torch.empty(3, 3, 256, dtype=torch.float64)
    for ry in range(3):
        for rx in range(3):
            bias[ry, rx] = b3 + sum(btap[ky, kx] for ky in valid[ry] for kx in valid[rx])
    return _conv_to_nk(Wc), bias.reshape(9, 256)


# bilinear x2 (align_corners=False) as a 1-D operator: hi-res sample 2j + p + (k - 1), k = conv tap 0..2, is a blend of the
# low-res samples j-1, j, j+1 with these weights (interior; the two outermost hi-res rows / columns differ and are recomputed
# by conv1_ring_kernel).  _UP2[p][k][l + 1]
_UP2 = torch.tensor([[[0.75, 0.25, 0.0], [0.25, 0.75, 0.0], [0.0, 0.75, 0.25]],
                     [[0.25, 0.75, 0.0], [0.0, 0.75, 0.25], [0.0, 0.25, 0.75]]], dtype=torch.float64)


def _compose_up2_conv3(w):
    """conv3x3(pad 1) o bilinear-x2 == four 3x3 convolutions on the LOW-res grid, one per output phase (py, px):
    [Cout, Cin, 3, 3] -> [4*Cout, Cin, 3, 3] with row = (py*2 + px)*Cout + o  (persformer_heads decoder: F.interpolate
    scale_factor=2 followed by conv_fuse_conv1, gravity_head.py:171-173 / latitude_head.py:170-172)."""
    w = w.double()
    return torch.cat([torch.einsum("oikm,kl,mn->oiln", w, _UP2[py], _UP2[px]) for py in (0, 1) for px in (0, 1)], 0)


def repack(sd, cfg):
    """sd: reference-layout state dict (CPU tensors).  cfg: entry of variants.VARIANTS."""
    out = {}
    bb = "backbone."
    # ---- the two 7x7 stems as [64][160] GEMM weights (K = (ky,kx,c) padded 147 -> 160 with zeros); ll_enc with its BatchNorm folded in
    scale = sd["ll_enc.bn1.weight"].double() / torch.sqrt(sd["ll_enc.bn1.running_var"].double() + 1e-5)
    llenc_b = sd["ll_enc.bn1.bias"].double() - sd["ll_enc.bn1.running_mean"].double() * scale
    for name, w, b in (("embed1g", sd[bb + "patch_embed1.proj.weight"].double(), sd[bb + "patch_embed1.proj.bias"]),
                       ("llencg", sd["ll_enc.conv1.weight"].double() * scale[:, None, None, None], llenc_b)):
        wk = torch.zeros(64, 160, dtype=torch.float64)
        wk[:, :147] = w.permute(0, 2, 3, 1).reshape(64, 147)
        _put_gemm(out, name, wk, b)
    # ---- MiT-B3
    for s, C in enumerate(MIT_DIMS):
        _put_ln(out, f"embed{s + 1}.ln", sd, f"{bb}patch_embed{s + 1}.norm")
        if s > 0:
            _put_gemm(out, f"embed{s + 1}", _conv_to_nk(sd[f"{bb}patch_embed{s + 1}.proj.weight"]), sd[f"{bb}patch_embed{s + 1}.proj.bias"])
        for i in range(MIT_DEPTHS[s]):
            k = f"{bb}block{s + 1}.{i}."
            n = f"s{s + 1}.b{i}."
            _put_ln(out, n + "ln1", sd, k + "norm1")
            _put_gemm(out, n + "q", sd[k + "attn.q.weight"], sd[k + "attn.q.bias"])
            if MIT_SR[s] > 1:
                _put_gemm(out, n + "sr", _conv_to_nk(sd[k + "attn.sr.weight"]), sd[k + "attn.sr.bias"])
                _put_ln(out, n + "srln", sd, k + "attn.norm")
            _put_gemm(out, n + "kv", sd[k + "attn.kv.weight"], sd[k + "attn.kv.bias"])
            _put_gemm(out, n + "proj", sd[k + "attn.proj.weight"], sd[k + "attn.proj.bias"])
            _put_ln(out, n + "ln2", sd, k + "norm2")
            _put_gemm(out, n + "fc1", sd[k + "mlp.fc1.weight"], sd[k + "mlp.fc1.bias"])
            dw = sd[k + "mlp.dwconv.dwconv.weight"]
            out[n + "dw.w"] = dw.reshape(dw.shape[0], 9).t().float().contiguous()
            out[n + "dw.b"] = sd[k + "mlp.dwconv.dwconv.bias"].float().contiguous()
            _put_gemm(out, n + "fc2", sd[k + "mlp.fc2.weight"], sd[k + "mlp.fc2.bias"])
        _put_ln(out, f"s{s + 1}.norm", sd, f"{bb}norm{s + 1}")
    # ---- decoder heads (group 0 = gravity, group 1 = latitude)
    heads = ("gravity_head", "latitude_head")
    for lvl in (1, 2, 3, 4):
        ws, bs = zip(*(_compose_proc(sd, h, lvl) for h in heads))
        _put_gemm(out, f"head.proc{lvl}", torch.cat(ws, 0), torch.cat(bs, 1).reshape(-1))   # [512, 9C], [9*512]
    for f in (1, 2, 3, 4):
        for u in (1, 2):
            if f == 4 and u == 1:
                continue
            for c in (1, 2):
                ks = [f"persformer_heads.{h}.fusion{f}.resConfUnit{u}.conv{c}" for h in heads]
                _put_gemm(out, f"head.f{f}.u{u}.c{c}", torch.stack([_conv_to_nk(sd[k + ".weight"]) for k in ks]),
                          torch.stack([sd[k + ".bias"] for k in ks]).reshape(-1))
    ks = [f"persformer_heads.{h}.conv_fuse_conv0.conv" for h in heads]
    _put_gemm(out, "head.conv0", torch.stack([_conv_to_nk(sd[k + ".weight"]) for k in ks]), torch.stack([sd[k + ".bias"] for k in ks]).reshape(-1))
    # conv_fuse_conv1 composed with the x2 upsample in front of it: N = 4 phases x 32 per head on the 160x160 grid; plus the
    # plain fp32 weights as [head][tap][ci][o] for the border-ring kernel
    ks = [f"persformer_heads.{h}.conv_fuse_conv1.conv" for h in heads]
    _put_gemm(out, "head.conv1p", torch.stack([_conv_to_nk(_compose_up2_conv3(sd[k + ".weight"])) for k in ks]),
              torch.stack([sd[k + ".bias"].repeat(4) for k in ks]).reshape(-1))
    out["head.conv1f.w"] = torch.stack([sd[k + ".weight"].permute(2, 3, 1, 0).reshape(9, 64, 32) for k in ks]).float().contiguous()
    out["head.conv1f.b"] = torch.stack([sd[k + ".bias"] for k in ks]).reshape(-1).float().contiguous()
    for short, h, pred in (("g", "gravity_head", "linear_pred_gravity"), ("l", "latitude_head", "linear_pred_latitude")):
        w = sd[f"persformer_heads.{h}.{pred}.weight"]
        out[f"head.pred_{short}.w"] = w.reshape(w.shape[0], 32).float().contiguous()
        out[f"head.pred_{short}.b"] = sd[f"persformer_heads.{h}.{pred}.bias"].float().contiguous()
    # ---- ParamNet (ConvNeXt-T)
    if cfg["param_net"] is not None:
        repack_param_net(sd, out)
    return out


PN = "param_net.backbone."


def repack_param_net(sd, out):
    """The ParamNet part of ``repack``: ``sd``'s ``param_net.backbone.*`` tensors (any device) -> ``out[name]`` on the same device.
    ``PerspectiveFields`` also runs it on the device, on its trainable ParamNet parameters."""
    pn = PN
    out["pn.stem.w"] = _stem(sd[pn + "downsample_layers.0.0.weight"])
    out["pn.stem.b"] = sd[pn + "downsample_layers.0.0.bias"].float().contiguous()
    _put_ln(out, "pn.stem.ln", sd, pn + "downsample_layers.0.1")
    for k in (1, 2, 3):
        _put_ln(out, f"pn.ds{k}.ln", sd, f"{pn}downsample_layers.{k}.0")
        _put_gemm(out, f"pn.ds{k}", _conv_to_nk(sd[f"{pn}downsample_layers.{k}.1.weight"]), sd[f"{pn}downsample_layers.{k}.1.bias"])
    for s, C in enumerate(CNX_DIMS):
        for j in range(CNX_DEPTHS[s]):
            k = f"{pn}stages.{s}.{j}."
            n = f"pn.s{s}.b{j}."
            dw = sd[k + "dwconv.weight"]
            out[n + "dw.w"] = dw.reshape(C, 49).t().float().contiguous()
            out[n + "dw.b"] = sd[k + "dwconv.bias"].float().contiguous()
            _put_ln(out, n + "ln", sd, k + "norm")
            _put_gemm(out, n + "pw1", sd[k + "pwconv1.weight"], sd[k + "pwconv1.bias"])
            _put_gemm(out, n + "pw2", sd[k + "pwconv2.weight"], sd[k + "pwconv2.bias"])
            out[n + "gamma"] = sd[k + "gamma"].float().contiguous()
    _put_ln(out, "pn.norm", sd, pn + "norm")
    out["pn.head.w"] = sd[pn + "head.weight"].float().contiguous()
    out["pn.head.b"] = sd[pn + "head.bias"].float().contiguous()
    return out


def param_net_train_weights(sd, out):
    """The extra engine tensors of ParamNet's backward (pf_param_backward): the transposed hi / lo planes of every GEMM weight
    (data gradients dX = dY W run on the GEMM engine as dY (W^T)^T), the depthwise kernels rotated by 180 degrees (their data
    gradient is the forward kernel with the rotated weights) and a zero bias for that launch."""
    pn = PN
    for k in (1, 2, 3):
        hi, lo = split_hi_lo(_conv_to_nk(sd[f"{pn}downsample_layers.{k}.1.weight"]).t())
        out[f"pn.ds{k}.t.whi"], out[f"pn.ds{k}.t.wlo"] = hi, lo
    for s, C in enumerate(CNX_DIMS):
        for j in range(CNX_DEPTHS[s]):
            k = f"{pn}stages.{s}.{j}."
            n = f"pn.s{s}.b{j}."
            for short, key in (("pw1t", "pwconv1"), ("pw2t", "pwconv2")):
                out[n + short + ".whi"], out[n + short + ".wlo"] = split_hi_lo(sd[k + key + ".weight"].t())
            out[n + "dw.wr"] = sd[k + "dwconv.weight"].reshape(C, 49).flip(1).t().float().contiguous()
    ref = sd[pn + "norm.weight"]
    out["pn.zero"] = torch.zeros(768, dtype=torch.float32, device=ref.device)
    return out


def param_net_grad_to_ref(name, g):
    """A gradient in the engine layout of ``name`` (pf_param_grad_entry) -> (reference key, tensor in the reference's shape):
    the inverse of the permutes of ``repack_param_net``."""
    pn = PN
    parts = name.split(".")
    if name.startswith("pn.stem."):
        if name == "pn.stem.w":
            return pn + "downsample_layers.0.0.weight", g.view(4, 4, 3, 96).permute(3, 2, 0, 1)
        if name == "pn.stem.b":
            return pn + "downsample_layers.0.0.bias", g
        return pn + "downsample_layers.0.1." + {"w": "weight", "b": "bias"}[parts[-1]], g
    if name.startswith("pn.ds"):
        k = int(parts[1][2:])
        if parts[2] == "ln":
            return f"{pn}downsample_layers.{k}.0." + {"w": "weight", "b": "bias"}[parts[3]], g
        cout, cin = CNX_DIMS[k], CNX_DIMS[k - 1]
        if parts[2] == "w":
            return f"{pn}downsample_layers.{k}.1.weight", g.view(cout, 2, 2, cin).permute(0, 3, 1, 2)
        return f"{pn}downsample_layers.{k}.1.bias", g
    if name.startswith("pn.norm."):
        return pn + "norm." + {"w": "weight", "b": "bias"}[parts[-1]], g
    if name.startswith("pn.head."):
        return pn + "head." + {"w": "weight", "b": "bias"}[parts[-1]], g.view(5, 768) if parts[-1] == "w" else g
    s, j = int(parts[1][1:]), int(parts[2][1:])
    C = CNX_DIMS[s]
    k = f"{pn}stages.{s}.{j}."
    leaf = ".".join(parts[3:])
    if leaf == "dw.w":
        return k + "dwconv.weight", g.view(49, C).t().reshape(C, 1, 7, 7)
    if leaf == "dw.b":
        return k + "dwconv.bias", g
    if leaf == "gamma":
        return k + "gamma", g
    layer, wb = parts[3], parts[4]
    if layer == "ln":
        return k + "norm." + {"w": "weight", "b": "bias"}[wb], g
    key = {"pw1": "pwconv1", "pw2": "pwconv2"}[layer]
    if wb == "w":
        return k + key + ".weight", g.view(4 * C, C) if layer == "pw1" else g.view(C, 4 * C)
    return k + key + ".bias", g
