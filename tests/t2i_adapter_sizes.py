"""The production sizes of the T2I-Adapter tests, kept next to `production.py`'s tables: base UNet -> latent (h, w).
SD v1.5 at 512² and 512x768 (the adapter's 96/48/24/12-wide levels take the im2col A tile), SDXL at 1024² and
1216x832 (76x52 and 38x26); the adapter runs for 1 image and the engine's maximum of 8."""

T2I_ADAPTER_SIZES = {
    "sd15": ((64, 64), (64, 96)),
    "sdxl": ((128, 128), (152, 104)),
}
T2I_ADAPTER_BATCHES = (1, 8)
