"""Where a diffusers-format pipeline directory keeps the files the native components load — the layout
`StableDiffusionPipeline.from_pretrained` / `StableDiffusionXLPipeline.from_pretrained` read in the reference
(latent_diffusion.py:62-66, latent_sdxl.py:41-49):

    <dir>/unet/diffusion_pytorch_model[.fp16].safetensors
    <dir>/vae/diffusion_pytorch_model[.fp16].safetensors        (SDXL: the reference swaps in madebyollin/sdxl-vae-fp16-fix)
    <dir>/text_encoder/model[.fp16].safetensors      + <dir>/tokenizer/{vocab.json, merges.txt}
    <dir>/text_encoder_2/model[.fp16].safetensors    + <dir>/tokenizer_2/{vocab.json, merges.txt}     (SDXL only)

The SDXL refiner (family 'sdxl_refiner') has unet/, vae/, text_encoder_2/ and tokenizer_2/ only: no text_encoder/.

SD 2.x (family 'sd20') has the SD v1.5 layout; its text_encoder is OpenCLIP ViT-H. `scheduler/scheduler_config.json`
(prediction_type) and `unet/config.json` (sample_size) are read when present, so the 768^2 v-prediction checkpoints
(stable-diffusion-2, -2-1) and the 512^2 epsilon ones (-2-base, -2-1-base) both load with the right UNet config.

`solver_components(dir, family, device)` turns it into the keyword arguments of `get_solver(...)`. Nothing can be
downloaded here; without a directory every component falls back to seeded synthetic weights."""
from __future__ import annotations

import json
from pathlib import Path
from typing import Dict, Optional


def _weights(folder: Path, stems) -> Optional[Path]:
    for stem in stems:
        for name in (f"{stem}.fp16.safetensors", f"{stem}.safetensors"):
            if (folder / name).is_file():
                return folder / name
    return None


def find_pipeline_files(ckpt_dir, family: str) -> Dict[str, Path]:
    """family: 'sd15' | 'sd20' | 'sdxl' | 'sdxl_refiner'. Raises FileNotFoundError naming every missing piece. For 'sd20'
    the optional config files are included as 'scheduler_config' / 'unet_config' when they exist."""
    root = Path(ckpt_dir)
    want = {"unet": (root / "unet", ("diffusion_pytorch_model",)), "vae": (root / "vae", ("diffusion_pytorch_model",)),
            "text_encoder": (root / "text_encoder", ("model",))}
    toks = ["tokenizer"]
    if family in ("sdxl", "sdxl_refiner"):
        want["text_encoder_2"] = (root / "text_encoder_2", ("model",))
        toks.append("tokenizer_2")
        if family == "sdxl_refiner":  # the refiner has one text tower, OpenCLIP bigG
            del want["text_encoder"]
            toks.remove("tokenizer")
    elif family not in ("sd15", "sd20"):
        raise ValueError(f"unknown model family {family!r}")
    found: Dict[str, Path] = {}
    missing = []
    for key, (folder, stems) in want.items():
        p = _weights(folder, stems)
        if p is None:
            missing.append(f"{folder}/{stems[0]}[.fp16].safetensors")
        else:
            found[key] = p
    for t in toks:
        for name in ("vocab.json", "merges.txt"):
            p = root / t / name
            if p.is_file():
                found[f"{t}/{name}"] = p
            else:
                missing.append(str(p))
    if missing:
        raise FileNotFoundError("pipeline directory is incomplete, missing: " + ", ".join(missing))
    if family == "sd20":
        for key, p in (("scheduler_config", root / "scheduler" / "scheduler_config.json"),
                       ("unet_config", root / "unet" / "config.json")):
            if p.is_file():
                found[key] = p
    return found


def sd2_unet_config(files: Dict[str, Path]):
    """The SD 2 UNet config of a pipeline directory: 768^2 v-prediction unless scheduler_config.json / unet/config.json
    say otherwise (prediction_type, sample_size)."""
    from .config import sd2_config
    pred, size = "v_prediction", 96
    if "scheduler_config" in files:
        pred = json.loads(files["scheduler_config"].read_text()).get("prediction_type", "epsilon")
    if "unet_config" in files:
        size = int(json.loads(files["unet_config"].read_text()).get("sample_size", size))
    return sd2_config(sample_size=size, prediction_type=pred)


def solver_components(ckpt_dir, family: str, device) -> dict:
    """Keyword arguments for `latent_sdxl.get_solver` / `latent_diffusion.get_solver` that load every component of the
    pipeline directory on the native backend (UNet, VAE encoder + decoder, CLIP text towers + BPE tokenizers)."""
    from .text_encoder import get_conditioner
    from .vae import get_vae
    f = find_pipeline_files(ckpt_dir, family)
    kw = {"model_key": str(f["unet"])}
    if family == "sdxl":
        kw["vae"] = get_vae("sdxl_vae", device, str(f["vae"]))
        kw["text_encoders"] = (
            get_conditioner("clip_l", device, "sdxl", str(f["text_encoder"]), str(f["tokenizer/vocab.json"]),
                            str(f["tokenizer/merges.txt"])),
            get_conditioner("clip_bigg", device, "sdxl", str(f["text_encoder_2"]), str(f["tokenizer_2/vocab.json"]),
                            str(f["tokenizer_2/merges.txt"])))
    else:
        kw["vae"] = get_vae("sd15_vae", device, str(f["vae"]))
        kw["text_encoder"] = get_conditioner("clip_h" if family == "sd20" else "clip_l", device, "sd15",
                                             str(f["text_encoder"]), str(f["tokenizer/vocab.json"]),
                                             str(f["tokenizer/merges.txt"]))
        if family == "sd20":
            kw["unet_config"] = sd2_unet_config(f)
    return kw


def refiner_components(ckpt_dir, device) -> dict:
    """Keyword arguments for `latent_sdxl.SDXLRefiner` from an SDXL refiner pipeline directory: its UNet and its bigG
    text tower. Its VAE is the SDXL VAE the base solver already holds, so it is not loaded again."""
    from .text_encoder import get_conditioner
    f = find_pipeline_files(ckpt_dir, "sdxl_refiner")
    return {"model_key": str(f["unet"]),
            "text_encoder": get_conditioner("clip_bigg", device, "sdxl", str(f["text_encoder_2"]),
                                            str(f["tokenizer_2/vocab.json"]), str(f["tokenizer_2/merges.txt"]))}


def _model_dir_files(ckpt_dir, what: str) -> Dict[str, Path]:
    """{'config': <dir>/config.json, 'weights': <dir>/diffusion_pytorch_model[.fp16].safetensors} of a diffusers model
    directory. Raises FileNotFoundError naming every missing file."""
    root = Path(ckpt_dir)
    found: Dict[str, Path] = {}
    missing = []
    if (root / "config.json").is_file():
        found["config"] = root / "config.json"
    else:
        missing.append(f"{root}/config.json")
    w = _weights(root, ("diffusion_pytorch_model",))
    if w is None:
        missing.append(f"{root}/diffusion_pytorch_model[.fp16].safetensors")
    else:
        found["weights"] = w
    if missing:
        raise FileNotFoundError(f"{what} directory is missing: " + ", ".join(missing))
    return found


def find_controlnet_files(ckpt_dir) -> Dict[str, Path]:
    """A diffusers ControlNetModel directory: {'config': <dir>/config.json, 'weights':
    <dir>/diffusion_pytorch_model[.fp16].safetensors}. Raises FileNotFoundError naming every missing file."""
    return _model_dir_files(ckpt_dir, "ControlNet")


def find_t2i_adapter_files(ckpt_dir) -> Dict[str, Path]:
    """A diffusers T2IAdapter directory (e.g. TencentARC/t2iadapter_canny_sd15v2), laid out as find_controlnet_files'."""
    return _model_dir_files(ckpt_dir, "T2I-Adapter")
