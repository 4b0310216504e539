"""Generate tests/golden/wan_vae_stream_tiny.pt by running the REFERENCE's own chunked, feature-cached Wan VAE decode and encode
(/root/reference/wan23/modules/vae2_2.py and /root/reference/wan/modules/vae.py, `WanVAE_.decode` / `WanVAE_.encode`) on CPU at
reduced width on sequences long enough for several streamed chunks: a 9-latent-frame decode and 25- and 27-frame encodes per VAE
(27 is not 1 + 4k: the reference encodes its first 25 frames). The weights are the tiny fixtures' (same seeds and configs as
tools/make_golden_vae2{2,1}.py and make_golden_vae2{2,1}_enc.py). Authoring container only."""
from __future__ import annotations

import importlib.util
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
from oracle import wan21vae, wan21vae_enc, wan22vae, wan22vae_enc  # noqa: E402

MULT, NRB, TUP = (1, 2, 4, 4), 2, (True, True, False)
VAES = {
    # name: (reference file, decoder oracle, decoder cfg, decoder seed, encoder oracle, encoder cfg, encoder seed, decode HxW, encode HxW)
    "wan22": ("/root/reference/wan23/modules/vae2_2.py", wan22vae, dict(dec_dim=32, z_dim=16, dim_mult=MULT, num_res_blocks=NRB,
              temperal_upsample=TUP), 777, wan22vae_enc, dict(dim=32, z_dim=16, dim_mult=MULT, num_res_blocks=NRB,
              temperal_downsample=TUP[::-1]), 779, (4, 6), (32, 48)),
    "wan21": ("/root/reference/wan/modules/vae.py", wan21vae, dict(dim=32, z_dim=16, dim_mult=MULT, num_res_blocks=NRB,
              temperal_upsample=TUP), 778, wan21vae_enc, dict(dim=32, z_dim=16, dim_mult=MULT, num_res_blocks=NRB,
              temperal_downsample=TUP[::-1]), 780, (4, 6), (16, 24)),
}


@torch.no_grad()
def main():
    torch.set_num_threads(8)
    gold = {}
    for k, (name, (src, dmod, dcfg, dseed, emod, ecfg, eseed, dhw, ehw)) in enumerate(VAES.items()):
        spec = importlib.util.spec_from_file_location(f"ref_{name}", src)
        ref = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(ref)
        sd = {**dmod.make_state_dict(dseed, **dcfg), **emod.make_state_dict(eseed, **ecfg)}
        kw = dict(dim=32, dec_dim=32) if name == "wan22" else dict(dim=32)
        model = ref.WanVAE_(z_dim=16, dim_mult=list(MULT), num_res_blocks=NRB, attn_scales=[],
                            temperal_downsample=list(TUP[::-1]), **kw)
        model.load_state_dict(sd, strict=True)
        model.eval()
        g = torch.Generator().manual_seed(40 + k)
        mean, std = 0.3 * torch.randn(16, generator=g), 0.5 + torch.rand(16, generator=g)
        scale = [mean, 1.0 / std]
        z = torch.randn(16, 9, *dhw, generator=torch.Generator().manual_seed(900 + k))
        out = model.decode(z.unsqueeze(0), scale).float().clamp_(-1, 1).squeeze(0)
        entry = {"dec_cfg": dcfg, "dec_seed": dseed, "enc_cfg": ecfg, "enc_seed": eseed, "mean": mean, "std": std,
                 "decode": dict(seed=900 + k, T=9, H=dhw[0], W=dhw[1], shape=tuple(out.shape), sample=out[..., ::3, ::3].clone(),
                                rowsum=out.sum(-1), colsum=out.sum(-2)), "encode": {}}
        print(name, "decode", tuple(out.shape))
        for T in (25, 27):
            x = torch.randn(3, T, *ehw, generator=torch.Generator().manual_seed(950 + T + k)).clamp_(-1, 1)
            model.clear_cache()
            mu = model.encode(x.unsqueeze(0), scale).float().squeeze(0)
            entry["encode"][T] = dict(seed=950 + T + k, T=T, H=ehw[0], W=ehw[1], shape=tuple(mu.shape), mu=mu.clone())
            print(name, "encode", T, tuple(mu.shape))
        gold[name] = entry
    path = ROOT / "tests" / "golden" / "wan_vae_stream_tiny.pt"
    torch.save(gold, path)
    print(path.name, path.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
