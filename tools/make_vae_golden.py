"""TEST INFRASTRUCTURE — golden outputs of the reference's VAE at its real channel width. Writes
tests/golden/vae_full_width.pt from the UNMODIFIED reference `Decoder(post_quant_conv(z))` (autoencoder.py:362-365;
model.py:882-1030) and `quant_conv(Encoder(x))` (autoencoder.py:352-357; model.py:763-880).

tests/golden/vae_decode_small.pt (`python -m oracle.make_golden --only vae`) shrinks the ddconfig to ch 64, so its
mid-block attention is only 128 wide. This file keeps the inference config's ddconfig (configs/inference_nuscenes.yaml:
ch 128, ch_mult [1, 2, 4, 4], num_res_blocks 2: C = 512 in the mid block) and shrinks the picture instead:
z [2, 4, 8, 48] -> image [2, 3, 64, 384] and x [2, 3, 64, 384] -> moments [2, 8, 8, 48]. Weights and inputs are
re-derived from seeds (`vae_decoder_weights`, `full_width_inputs`), which tests import; the file stores the key lists
and the two reference outputs (about 0.6 MB).

Run where the reference tree is available:  python -m tools.make_vae_golden
"""
from __future__ import annotations

import contextlib
import io
import sys
from pathlib import Path

import torch

GOLDEN = Path(__file__).resolve().parent.parent / "tests" / "golden"
FULL_WIDTH_DDCONFIG = dict(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                           num_res_blocks=2, attn_resolutions=[], dropout=0.0)
DECODER_SEED, ENCODER_SEED = 31, 32


def full_width_inputs():
    """(z [2, 4, 8, 48], x [2, 3, 64, 384]): 2 frames, 6 views of 8 x 8 latents / 64 x 64 pixels."""
    g = torch.Generator(device="cpu").manual_seed(33)
    z = torch.randn(2, 4, 8, 48, generator=g)
    x = torch.rand(2, 3, 64, 384, generator=g) * 2.0 - 1.0
    return z, x


@torch.no_grad()
def golden_vae_full_width() -> dict:
    from oracle import ref_loader as R
    from oracle.make_golden import vae_decoder_weights
    from panacea_b200.vae import decoder_param_spec, encoder_param_spec
    R.import_reference()
    from sgm.modules.diffusionmodules import model as M
    dd = FULL_WIDTH_DDCONFIG
    z, x = full_width_inputs()
    spec = decoder_param_spec(dd, 4)
    sd = vae_decoder_weights(spec, seed=DECODER_SEED)
    with contextlib.redirect_stdout(io.StringIO()):
        dec = M.Decoder(**dd).eval()
    dec.load_state_dict({k[len("decoder."):]: v for k, v in sd.items() if k.startswith("decoder.")}, strict=True)
    pq = torch.nn.Conv2d(4, 4, 1)
    pq.load_state_dict({"weight": sd["post_quant_conv.weight"], "bias": sd["post_quant_conv.bias"]})
    image = dec(pq(z))
    espec = encoder_param_spec(dd, 4)
    esd = vae_decoder_weights(espec, seed=ENCODER_SEED)
    with contextlib.redirect_stdout(io.StringIO()):
        enc = M.Encoder(**dd).eval()
    enc.load_state_dict({k[len("encoder."):]: v for k, v in esd.items() if k.startswith("encoder.")}, strict=True)
    qc = torch.nn.Conv2d(8, 8, 1)
    qc.load_state_dict({"weight": esd["quant_conv.weight"], "bias": esd["quant_conv.bias"]})
    moments = qc(enc(x))
    return {"ddconfig": dd, "decoder_seed": DECODER_SEED, "encoder_seed": ENCODER_SEED, "keys": sorted(spec),
            "encoder_keys": sorted(espec), "image": image.contiguous(), "moments": moments.contiguous()}


def main(argv=None):
    g = golden_vae_full_width()
    torch.save(g, GOLDEN / "vae_full_width.pt")
    print(f"vae_full_width.pt image {tuple(g['image'].shape)} rms={g['image'].pow(2).mean().sqrt():.4f} "
          f"moments {tuple(g['moments'].shape)} rms={g['moments'].pow(2).mean().sqrt():.4f}")


if __name__ == "__main__":
    main(sys.argv[1:])
