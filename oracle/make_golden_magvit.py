"""Pins oracle/magvit.py against the REAL MAGVITv2 decoder (imported read-only from MMDP_REFERENCE_ROOT) and writes
tests/golden/magvit_decode.pt. Needs MMDP_REFERENCE_ROOT.    PYTHONDONTWRITEBYTECODE=1 python -m oracle.make_golden_magvit"""
import contextlib
import io
import os

import torch

from . import magvit, ref_shim

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")


def main():
    torch.set_num_threads(8)
    _, _, mv = ref_shim.load_m()
    assert mv is not None, "reference modeling_magvitv2 could not be imported"
    out = {}
    # (1) reduced decoder (fast; also exercised by the CPU test-suite): 2 levels, ch 32
    small = magvit.decoder_config(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 2))
    # (2) the real default decoder (39.9 M parameters, 1.2 TFLOP per 1024-token image)
    full = magvit.decoder_config()
    for tag, cfg, seed, n_tok, batch in (("small", small, 3, 64, 2), ("full", full, 4, 1024, 1)):
        w = magvit.make_weights(cfg, seed)
        with contextlib.redirect_stdout(io.StringIO()):
            dec = mv.VQGANDecoder(ch=cfg.ch, ch_mult=list(cfg.ch_mult), num_res_blocks=list(cfg.num_res_blocks),
                                  z_channels=cfg.z_channels).eval()
            lfq = mv.LFQuantizer(codebook_dim=13)
        missing, unexpected = dec.load_state_dict({k[len("decoder."):]: v for k, v in w.items()}, strict=True)
        idx = torch.randint(0, 8192, (batch, n_tok), generator=torch.Generator().manual_seed(seed + 100))
        with torch.no_grad():
            ref = dec(lfq.get_codebook_entry(idx))["output"]          # == MAGVITv2.decode_code
        got = magvit.decode_code(idx, w, cfg)
        assert torch.equal(ref, got), f"oracle decoder != reference decoder ({tag})"
        s = 1 if tag == "small" else 8
        out[tag] = dict(cfg=dict(ch=cfg.ch, ch_mult=cfg.ch_mult, num_res_blocks=cfg.num_res_blocks), weight_seed=seed, idx=idx,
                        stride=s, image=ref[:, :, ::s, ::s].clone(), mean=float(ref.mean()), std=float(ref.std()),
                        absmax=float(ref.abs().max()), shape=tuple(ref.shape))
        print(tag, "ok", tuple(ref.shape), "std", float(ref.std()), "absmax", float(ref.abs().max()))
    torch.save(out, os.path.join(OUT, "magvit_decode.pt"))

    # ---- encoder: MAGVITv2.get_code -------------------------------------------------------------------------
    enc_out = {}
    small_e = magvit.encoder_config(ch=32, ch_mult=(1, 2), num_res_blocks=(1, 2))
    full_e = magvit.encoder_config()
    for tag, cfg, seed, res, batch in (("small", small_e, 13, 32, 2), ("full", full_e, 14, 512, 1)):
        w = magvit.make_encoder_weights(cfg, seed)
        with contextlib.redirect_stdout(io.StringIO()):
            enc = mv.VQGANEncoder(ch=cfg.ch, ch_mult=list(cfg.ch_mult), num_res_blocks=list(cfg.num_res_blocks), z_channels=cfg.z_channels).eval()
            lfq = mv.LFQuantizer(codebook_dim=13)
        enc.load_state_dict({k[len("encoder."):]: v for k, v in w.items()}, strict=True)
        px = torch.rand(batch, 3, res, res, generator=torch.Generator().manual_seed(seed + 100)) * 2 - 1
        with torch.no_grad():
            z_ref = enc(px)
            ids_ref = lfq.get_indices(lfq(z_ref)["z"]).reshape(batch, -1)          # == MAGVITv2.get_code
        z = magvit.encoder_forward(px, w, cfg)
        assert torch.equal(z_ref, z), f"oracle encoder != reference encoder ({tag})"
        assert torch.equal(ids_ref, magvit.get_code(px, w, cfg)), f"oracle get_code != reference ({tag})"
        enc_out[tag] = dict(cfg=dict(ch=cfg.ch, ch_mult=cfg.ch_mult, num_res_blocks=cfg.num_res_blocks), weight_seed=seed,
                            pixel_seed=seed + 100, res=res, batch=batch, z=z_ref.clone(), ids=ids_ref.clone())
        print("encoder", tag, "ok", tuple(z_ref.shape), "z std", float(z_ref.std()))
    torch.save(enc_out, os.path.join(OUT, "magvit_encode.pt"))


if __name__ == "__main__":
    main()
