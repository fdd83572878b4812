#!/usr/bin/env python
"""VQGAN ends at the BASELINE configs[2] shape (LBBDM-f4: images [B,3,256,256] <-> latents [B,3,64,64], ch 128,
mult (1,2,4), 8192 codes): VQGANEngine (split-bf16 x3, fp32-class) vs the same graph on the PyTorch library path
(fp32 / TF32 / bf16 autocast).  One encode = what LatentBrownianBridgeModel.encode costs (twice per training
sample, once per sampled batch); one decode = quantize + post_quant_conv + decoder.

    python tools/bench_vqgan.py [B]                                  the f4 table above (B = 32)
    python tools/bench_vqgan.py --size 224 --template f8 [--batch 4]  one template autoencoder at one image size:
        native encode / decode against the module path the latent model otherwise takes (the same graph in stock
        PyTorch with torch's default TF32 convolutions), with the card's name and power limit"""
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bbdm_b200.vqgan import VQModel  # noqa: E402

DD = dict(double_z=False, z_channels=3, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=(1, 2, 4),
          num_res_blocks=2, attn_resolutions=[], dropout=0.0)
# Template-LBBDM-f4 / f8 / f16 autoencoders: (ddconfig, n_embed, embed_dim)
TEMPLATES = {
    "f4": (DD, 8192, 3),
    "f8": (dict(DD, z_channels=4, ch_mult=(1, 2, 2, 4), attn_resolutions=[32]), 16384, 4),
    "f16": (dict(DD, z_channels=16, ch_mult=(1, 1, 2, 2, 4), attn_resolutions=[16]), 16384, 16),
}


# ---- stock-PyTorch forward of the same parameter tree (library baseline only) ------------------------------
def gn(m, x):
    return F.group_norm(x, 32, m.weight, m.bias, 1e-6)


def resnet(m, x):
    h = m.conv1(F.silu(gn(m.norm1, x)))
    h = m.conv2(F.silu(gn(m.norm2, h)))
    if hasattr(m, "nin_shortcut"):
        x = m.nin_shortcut(x)
    return x + h


def attn(m, x):
    b, c, hh, ww = x.shape
    h = gn(m.norm, x)
    q, k, v = (f(h).reshape(b, c, -1) for f in (m.q, m.k, m.v))
    w = torch.softmax(torch.bmm(q.transpose(1, 2), k) * (c ** -0.5), dim=2)
    return x + m.proj_out(torch.bmm(v, w.transpose(1, 2)).reshape(b, c, hh, ww))


def mid(m, h):
    return resnet(m.block_2, attn(m.attn_1, resnet(m.block_1, h)))


def lib_encode(vq, x):
    e = vq.encoder
    h = e.conv_in(x)
    for i in range(e.num_resolutions):
        for j, blk in enumerate(e.down[i].block):
            h = resnet(blk, h)
            if len(e.down[i].attn) > 0:
                h = attn(e.down[i].attn[j], h)
        if i != e.num_resolutions - 1:
            h = e.down[i].downsample.conv(F.pad(h, (0, 1, 0, 1)))
    return vq.quant_conv(e.conv_out(F.silu(gn(e.norm_out, mid(e.mid, h)))))


def lib_decode(vq, z, idx=None, return_idx=False):
    cb = vq.quantize.embedding.weight
    zf = z.permute(0, 2, 3, 1).reshape(-1, cb.shape[1]).float()
    if idx is None:
        d = (zf ** 2).sum(1, keepdim=True) + (cb ** 2).sum(1) - 2 * zf @ cb.t()
        idx = d.argmin(1)
    if return_idx:
        return idx
    zq = cb[idx.reshape(-1)].view(z.shape[0], z.shape[2], z.shape[3], -1).permute(0, 3, 1, 2)
    dcd = vq.decoder
    h = mid(dcd.mid, dcd.conv_in(vq.post_quant_conv(zq)))
    for i in reversed(range(dcd.num_resolutions)):
        for j, blk in enumerate(dcd.up[i].block):
            h = resnet(blk, h)
            if len(dcd.up[i].attn) > 0:
                h = attn(dcd.up[i].attn[j], h)
        if i != 0:
            h = dcd.up[i].upsample.conv(F.interpolate(h, scale_factor=2.0, mode="nearest"))
    return dcd.conv_out(F.silu(gn(dcd.norm_out, h)))


def timeit(fn, steps=5, warmup=2):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def make_vq(template):
    dd, n_embed, embed_dim = TEMPLATES[template]
    torch.manual_seed(0)
    vq = VQModel(ddconfig=dd, n_embed=n_embed, embed_dim=embed_dim).eval().cuda()
    with torch.no_grad():
        for n, p in vq.named_parameters():
            if p.dim() >= 2:
                p.normal_(0, 0.02)
        vq.quantize.embedding.weight.normal_(0, 0.5)
    return vq


def _arg(name, default):
    return type(default)(sys.argv[sys.argv.index(name) + 1]) if name in sys.argv else default


def size_mode():
    """One template autoencoder at one image size: native encode / decode vs the module path at torch's defaults."""
    size, template, B = _arg("--size", 256), _arg("--template", "f8"), _arg("--batch", 4)
    steps, warmup = _arg("--steps", 10), _arg("--warmup", 3)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    vq = make_vq(template)
    f = 2 ** (len(TEMPLATES[template][0]["ch_mult"]) - 1)
    x = (0.5 * torch.randn(B, 3, size, size, device="cuda")).clamp_(-1, 1)
    with torch.no_grad():
        eng = vq.engine()
        z = eng.encode(x)
        lat = z + 0.2 * torch.randn_like(z)
        native = {"encode_ms": timeit(lambda: eng.encode(x), steps, warmup),
                  "decode_ms": timeit(lambda: eng.decode(lat), steps, warmup)}
        module = {"encode_ms": timeit(lambda: lib_encode(vq, x), steps, warmup),
                  "decode_ms": timeit(lambda: lib_decode(vq, lat), steps, warmup)}
        dev = lambda a, b: float((a - b).abs().max() / b.abs().max())
        z_mod = lib_encode(vq, x)
    print(json.dumps({"what": f"VQGAN-{template} ends, images [{B},3,{size},{size}], attention map {size // f}^2 "
                              f"(T = {(size // f) ** 2})", "gpu": smi, "native split3": native,
                      "module path (torch defaults: cudnn.allow_tf32=%s)" % torch.backends.cudnn.allow_tf32: module,
                      "encode_rel_dev_native_vs_module": dev(z, z_mod)}))


def main():
    if "--size" in sys.argv:
        return size_mode()
    B = int(sys.argv[1]) if len(sys.argv) > 1 and sys.argv[1].isdigit() else 32
    vq = make_vq("f4")
    x = (0.5 * torch.randn(B, 3, 256, 256, device="cuda")).clamp_(-1, 1)
    rows = []
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False     # true-fp32 reference values
    with torch.no_grad():
        eng = vq.engine()
        z = eng.encode(x)
        lat = z + 0.2 * torch.randn_like(z)
        if "--profile" in sys.argv:            # one more pass of each end for an ncu launch list, nothing else
            eng.encode(x)
            eng.decode(lat)
            eng.decode(lat)
            torch.cuda.synchronize()
            return
        img, idx = eng.decode(lat, return_indices=True)
        # nearest-code ties at fp32 resolution may resolve differently in the two fp32 evaluations of d: report the
        # agreement, and compare the decoded images for identical codes
        agree = float((lib_decode(vq, lat, return_idx=True) == idx.reshape(-1)).float().mean())
        ref_z, ref_img = lib_encode(vq, x), lib_decode(vq, lat, idx=idx)
        dev = lambda a, b: float((a - b).abs().max() / b.abs().max())
        rows.append({"mode": "native split3", "encode_ms": timeit(lambda: eng.encode(x)), "decode_ms": timeit(lambda: eng.decode(lat)),
                     "encode_rel_dev_vs_fp32_library": dev(z, ref_z), "code_agreement_vs_fp32_library": agree,
                     "decode_rel_dev_vs_fp32_library_same_codes": dev(img, ref_img)})
        for mode in ("fp32", "tf32", "bf16"):
            torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = mode == "tf32"
            torch.backends.cudnn.benchmark = True
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=mode == "bf16"):
                rows.append({"mode": "library " + mode, "encode_ms": timeit(lambda: lib_encode(vq, x)),
                             "decode_ms": timeit(lambda: lib_decode(vq, lat)),
                             "encode_rel_dev_vs_fp32_library": dev(lib_encode(vq, x).float(), ref_z)})
    print(json.dumps({"what": "VQGAN-f4 ends, images [%d,3,256,256]; algorithmic GFLOP/img: encode 345, decode 671" % B,
                      "batch": B, "rows": rows}))


if __name__ == "__main__":
    main()
