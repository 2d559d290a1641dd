"""What the executors' weight store and plan workspaces promise beyond the numerics the parity tests check:
- a UNet is only built when every weight of its state dict is present: whichever key is missing, building the handle
  fails with `missing weight: <key>` (nothing on the Python side checks UNet keys);
- the VAE's reported workspace is the one of a decode of the prepared shape, whatever the encoder has planned."""
import re

import pytest
import torch

pytestmark = pytest.mark.gpu
dev = torch.device("cuda:0")


@pytest.mark.parametrize("name", ["tiny_sdxl", "tiny_sd15"])
def test_every_unet_weight_is_required(name):
    """One key per pattern (the key with its block / layer indices blanked) rather than all 620 / 686, each of which
    costs a handle: that still removes every weight suffix of every block family (down / mid / up, resnets with and
    without a shortcut, transformers, samplers, embeddings)."""
    from cfgpp_b200 import _native as nv, config as C, weights as Wt
    from cfgpp_b200.engine import NativeUNet
    cfg = C.CONFIGS[name]()
    full = Wt.synthetic_state_dict(cfg, seed=3, device=dev)
    patterns = {}
    for k in full:
        patterns.setdefault(re.sub(r"(?<=\.)\d+(?=\.)", "#", k), k)
    keys = list(patterns.values())
    wrong = []
    for key in keys:
        sd = {k: v for k, v in full.items() if k != key}
        try:
            NativeUNet(cfg, sd, dev)
        except nv.NativeError as e:
            if not str(e).endswith(f"missing weight: {key}"):
                wrong.append((key, str(e)))
        else:
            wrong.append((key, "built without it"))
    assert not wrong, f"{len(wrong)} of {len(keys)} keys: {wrong[:5]}"
    NativeUNet(cfg, full, dev).close()  # and the complete state dict builds


def test_vae_workspace_is_the_decode_plans():
    from cfgpp_b200 import vae as V
    cfg = V.tiny_vae_config()
    sd = V.synthetic_vae_state_dict(cfg, seed=5, device=dev, with_encoder=True)
    vae = V.NativeVAEDecoder(cfg, sd, dev)
    assert vae.has_encoder
    z = torch.randn(1, 4, 16, 16, device=dev)
    vae.decode(z)
    ws = vae.stats["workspace_bytes"]
    assert ws > 0
    vae.encode(torch.rand(1, 3, 128, 128, device=dev) * 2 - 1)
    assert vae.stats["workspace_bytes"] == ws
    vae.encode(torch.rand(2, 3, 256, 256, device=dev) * 2 - 1)
    assert vae.stats["workspace_bytes"] == ws
    vae.decode(torch.randn(2, 4, 32, 32, device=dev))  # a decode re-plan replaces it ...
    assert vae.stats["workspace_bytes"] > ws
    vae.decode(z)  # ... and planning the first shape again restores it
    assert vae.stats["workspace_bytes"] == ws
    vae.close()
    # the decode workspace does not depend on whether the handle also holds an encoder
    dec_only = V.NativeVAEDecoder(cfg, {k: v for k, v in sd.items() if not k.startswith(("encoder.", "quant_conv."))},
                                  dev)
    assert not dec_only.has_encoder
    dec_only.decode(z)
    assert dec_only.stats["workspace_bytes"] == ws
    dec_only.close()
