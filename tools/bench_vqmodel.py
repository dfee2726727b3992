"""Times the native aMUSEd VQ-VAE (mmada_parallel_b200.vqmodel.VQModel) at the aMUSEd 512 configuration: decode of one
32x32 latent grid (512x512 pixels), encode of one 512x512 image, and the nearest-code search of its 1024 latents, with
CUDA events after warm-up. TFLOP/s use operation counts computed from the shapes below (multiply-adds of every
convolution counted as 2 FLOP; GroupNorm, SiLU, resampling and the codebook gather not counted), not measured ones.

With --parent-lib PATH (a libmmdp.so built from another commit) it also decodes the same MagViT ids with both libraries,
checks that the images are bit-identical, and times the two MagViT decoders alternately.

    python tools/bench_vqmodel.py [--iters 20] [--warmup 3] [--parent-lib /path/to/libmmdp.so] [--json out.json]
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import amused as AM  # noqa: E402  (seeded synthetic weights)
from oracle import magvit as OM  # noqa: E402


def conv_flops(cfg, h: int, w: int):
    """(decode, encode) FLOP of one image with an h x w latent grid."""
    boc, L, lat, lpb = cfg.block_out_channels, len(cfg.block_out_channels), cfg.latent_channels, cfg.layers_per_block

    def conv(px, cout, cin, k):
        return 2.0 * px * cout * cin * k * k

    def res(px, cin, cout):
        return conv(px, cout, cin, 3) + conv(px, cout, cout, 3) + (conv(px, cout, cin, 1) if cin != cout else 0.0)

    def mid(px, c):
        f = 2 * res(px, c, c)
        if cfg.mid_block_add_attention:
            f += 4 * 2.0 * px * c * c + 2 * 2.0 * px * px * c
        return f

    n = h * w
    dec = conv(n, lat, lat, 1) + conv(n, boc[-1], lat, 3) + mid(n, boc[-1])
    cin = boc[-1]
    for i in range(L):
        px = n * 4 ** i
        cout = boc[L - 1 - i]
        dec += res(px, cin, cout) + lpb * res(px, cout, cout)
        cin = cout
        if i != L - 1:
            dec += conv(px * 4, cout, cout, 3)
    dec += conv(n * 4 ** (L - 1), cfg.out_channels, boc[0], 3)
    px = n * 4 ** (L - 1)
    enc = conv(px, boc[0], cfg.in_channels, 3)
    cin = boc[0]
    for i in range(L):
        px = n * 4 ** (L - 1 - i)
        enc += res(px, cin, boc[i]) + (lpb - 1) * res(px, boc[i], boc[i])
        cin = boc[i]
        if i != L - 1:
            enc += conv(px // 4, boc[i], boc[i], 3)  # stride 2 (the kernel evaluates it at stride 1 and picks: 4x this)
    enc += mid(n, boc[-1]) + conv(n, lat, boc[-1], 3) + conv(n, lat, lat, 1)
    return dec, enc


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        q = f"unavailable ({e})"
    return name, q


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class ParentMagvit:
    """The MagViT decoder of another build of libmmdp.so, through its C ABI (same mmdp_vqdec_* signatures)."""

    def __init__(self, path, cfg, w):
        from mmada_parallel_b200 import _lib
        self.lib = C.CDLL(path)
        vp = C.c_void_p
        self.lib.mmdp_vqdec_create.argtypes = [C.POINTER(_lib.VqDecConfig), C.POINTER(vp)]
        self.lib.mmdp_vqdec_set_weight.argtypes = [vp, C.c_char_p, vp, C.c_int64, vp]
        self.lib.mmdp_vqdec_decode.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, vp, vp]
        self.lib.mmdp_vqdec_destroy.argtypes = [vp]
        self.lib.mmdp_last_error.restype = C.c_char_p
        c = _lib.VqDecConfig()
        c.ch, c.n_levels, c.z_channels, c.out_ch, c.max_batch, c.latent_h, c.latent_w = cfg.ch, len(cfg.ch_mult), 13, 3, 1, 32, 32
        for i, (m, n) in enumerate(zip(cfg.ch_mult, cfg.num_res_blocks)):
            c.ch_mult[i], c.num_res_blocks[i] = m, n
        self.h = vp()
        self._check(self.lib.mmdp_vqdec_create(C.byref(c), C.byref(self.h)))
        for k, v in w.items():
            t = v.float().contiguous()
            self._check(self.lib.mmdp_vqdec_set_weight(self.h, k.encode(), t.data_ptr(), t.numel(), None))
        torch.cuda.synchronize()

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError(self.lib.mmdp_last_error().decode())

    def decode(self, ids, out):
        self._check(self.lib.mmdp_vqdec_decode(self.h, ids.data_ptr(), 1, 32, 32, out.data_ptr(),
                                               torch.cuda.current_stream().cuda_stream or None))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--parent-lib", default=None)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vqmodel needs a CUDA device"
    from mmada_parallel_b200.magvit import MAGVITv2
    from mmada_parallel_b200.vqmodel import VQModel

    name, power = card()
    res = dict(card=name, power_limit_and_max_sm_clock=power)
    cfg = AM.make_config()
    w = AM.make_weights(cfg, 23)
    m = VQModel(**dict(AM.AMUSED_CONFIG, down_block_types=("DownEncoderBlock2D",) * 5, up_block_types=("UpDecoderBlock2D",) * 5,
                       lookup_from_codebook=True))
    m.load_state_dict(w)
    dec_f, enc_f = conv_flops(cfg, 32, 32)
    ids = torch.randint(0, 8192, (1, 32, 32), generator=torch.Generator().manual_seed(0)).cuda()
    px = torch.rand(1, 3, 512, 512, generator=torch.Generator().manual_seed(1)).cuda()
    lat = m.encode(px).latents
    t_dec = time_ms(lambda: m.decode(ids, force_not_quantize=True, shape=(1, 32, 32, 64)), args.iters, args.warmup)
    t_enc = time_ms(lambda: m.encode(px), args.iters, args.warmup)
    t_nn = time_ms(lambda: m.quantize(lat), args.iters * 10, args.warmup)
    res.update(amused_decode_512_ms=t_dec, amused_decode_tflop=dec_f / 1e12, amused_decode_tflops_per_s=dec_f / t_dec / 1e9,
               amused_encode_512_ms=t_enc, amused_encode_tflop=enc_f / 1e12, amused_encode_tflops_per_s=enc_f / t_enc / 1e9,
               nearest_1024x8192x64_ms=t_nn, nearest_gflop_per_s=3 * 1024 * 8192 * 64 / t_nn / 1e6)

    if args.parent_lib:
        mcfg = OM.decoder_config()
        mw = OM.make_weights(mcfg, 4)
        mine = MAGVITv2(latent_hw=(32, 32))
        mine.load_state_dict(mw)
        par = ParentMagvit(args.parent_lib, mcfg, mw)
        mids = torch.randint(0, 8192, (1, 1024), generator=torch.Generator().manual_seed(2)).cuda()
        a = mine.decode_code(mids)
        b = torch.empty_like(a)
        par.decode(mids, b)
        torch.cuda.synchronize()
        res["magvit_bit_identical_to_parent"] = bool(torch.equal(a, b))
        ts = {"this": [], "parent": []}
        for _ in range(5):
            ts["this"].append(time_ms(lambda: mine.decode_code(mids), args.iters, 1))
            ts["parent"].append(time_ms(lambda: par.decode(mids, b), args.iters, 1))
        res["magvit_decode_ms_this"] = ts["this"]
        res["magvit_decode_ms_parent"] = ts["parent"]
    print(json.dumps(res))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
