"""CLI with the reference's flag surface (examples/text_to_img.py:14-24):
    python -m examples.text_to_img --model sdxl --method ddim_cfg++ --cfg_guidance 0.6 --NFE 50 --prompt "..."
Runs on the Hopper-native (sm_90a) backend. Without checkpoints (offline) the UNet weights are seeded synthetic and the
text encoder / VAE are stand-ins (cfgpp_b200/conditioning.py), so the PNG is only a plumbing check."""
import argparse
import warnings
from pathlib import Path
from types import SimpleNamespace

import torch

from cfgpp_b200.batching import draw_latents
from cfgpp_b200.checkpoints import refiner_components, solver_components
from cfgpp_b200.config import sd2_config
from cfgpp_b200.latent_diffusion import get_solver
from cfgpp_b200.latent_sdxl import SDXLRefiner, get_solver as get_solver_sdxl
from cfgpp_b200.utils.log_util import create_workdir, set_seed


def model_family(model: str) -> str:
    """The checkpoint family of a --model choice: sd15 | sd20 | sdxl (SDXL-Lightning has the SDXL layout)."""
    return {"sd15": "sd15", "sd20": "sd20", "sdxl": "sdxl", "sdxl_lightning": "sdxl"}[model]


def build_solver(model: str, method: str, solver_config, device, ckpt_dir=None):
    """get_solver for --model: the SDXL registry for sdxl*, the SD registry otherwise — with the SD 2 UNet config
    (768^2 v-prediction unless the checkpoint directory says otherwise), ViT-H text tower and VAE for sd20."""
    family = model_family(model)
    extra = solver_components(ckpt_dir, family, device) if ckpt_dir else {}
    if family == "sd20":
        extra.setdefault("unet_config", sd2_config())
    return (get_solver_sdxl if family == "sdxl" else get_solver)(method, solver_config=solver_config, device=device,
                                                                 **extra)


def build_refiner(device, ckpt_dir=None) -> SDXLRefiner:
    """The SDXL refiner from its pipeline directory, or on seeded synthetic weights (with a warning) without one."""
    if ckpt_dir:
        return SDXLRefiner(device=device, **refiner_components(ckpt_dir, device))
    warnings.warn("no --refiner_ckpt_dir given; the SDXL refiner runs on seeded synthetic UNet weights")
    return SDXLRefiner(model_key="synthetic:8765", device=device)


def main():
    parser = argparse.ArgumentParser(description="Latent Diffusion")
    parser.add_argument("--workdir", type=Path, default="examples/workdir/t2i")
    parser.add_argument("--device", type=str, default="cuda")
    parser.add_argument("--null_prompt", type=str, default="low quality,jpeg artifacts,blurry,poorly drawn,ugly,worst quality,")
    parser.add_argument("--prompt", type=str, default="")
    parser.add_argument("--cfg_guidance", type=float, default=7.5)
    parser.add_argument("--method", type=str, default='ddim_cfg++')
    parser.add_argument("--model", type=str, default='sd15', choices=["sd15", "sd20", "sdxl", "sdxl_lightning"])
    parser.add_argument("--NFE", type=int, default=50)
    parser.add_argument("--seed", type=int, default=42)
    parser.add_argument("--ckpt_dir", type=Path, default=None,
                        help="diffusers-format pipeline directory (unet/, vae/, text_encoder[_2]/, tokenizer[_2]/); "
                             "default: seeded synthetic weights (nothing can be downloaded here)")
    parser.add_argument("--height", type=int, default=None,
                        help="image height in pixels (default: the model's native size, 512 for SD v1.5, 768 for "
                             "SD 2.x, 1024 for SDXL); a multiple of 8 * 2^(UNet levels - 1), e.g. 1216 x 832 for an SDXL bucket")
    parser.add_argument("--width", type=int, default=None, help="image width in pixels (default: native size)")
    parser.add_argument("--denoising_end", type=float, default=None,
                        help="--model sdxl: hand the last (1 - F) of the schedule to the SDXL refiner (e.g. 0.8; "
                             "methods ddim, ddim_cfg++, dpm++_2m_cfgpp); default: the base model alone")
    parser.add_argument("--refiner_ckpt_dir", type=Path, default=None,
                        help="SDXL refiner pipeline directory (unet/, vae/, text_encoder_2/, tokenizer_2/); default: "
                             "seeded synthetic refiner weights")
    parser.add_argument("--lora", action="append", default=[], metavar="PATH[:SCALE]",
                        help="a UNet LoRA *.safetensors (diffusers / peft or kohya naming) merged at SCALE (default 1.0); "
                             "repeatable, up to 4 adapters per weight")
    parser.add_argument("--controlnet", type=str, default=None, metavar="DIR",
                        help="a diffusers ControlNetModel directory (config.json + diffusion_pytorch_model"
                             "[.fp16].safetensors), or a name for seeded synthetic weights")
    parser.add_argument("--control_image", type=Path, default=None,
                        help="the control map (canny, depth, ...) as an image file at exactly the output size")
    parser.add_argument("--controlnet_scale", type=float, default=1.0)
    parser.add_argument("--control_guidance_start", type=float, default=0.0)
    parser.add_argument("--control_guidance_end", type=float, default=1.0)
    parser.add_argument("--ip_adapter", type=str, default=None, metavar="PATH",
                        help="IP-Adapter checkpoint (.bin / .safetensors); any other name: seeded synthetic weights")
    parser.add_argument("--ip_adapter_image", type=Path, default=None, help="the reference image of --ip_adapter")
    parser.add_argument("--ip_adapter_scale", type=float, default=1.0)
    parser.add_argument("--image_encoder", type=Path, default=None, metavar="DIR",
                        help="the adapter's CLIP image encoder (config.json + model.safetensors); default: synthetic")
    parser.add_argument("--t2i_adapter", type=str, default=None, metavar="DIR",
                        help="a diffusers T2IAdapter directory (config.json + diffusion_pytorch_model"
                             "[.fp16].safetensors), or a name for seeded synthetic weights")
    parser.add_argument("--t2i_adapter_image", type=Path, default=None,
                        help="the adapter's conditioning map (sketch, canny, depth, ...) at exactly the output size; read "
                             "as grayscale for a 1-channel adapter, RGB otherwise")
    parser.add_argument("--adapter_conditioning_scale", type=float, default=1.0)
    parser.add_argument("--adapter_conditioning_factor", type=float, default=1.0)
    args = parser.parse_args()
    if (args.t2i_adapter is None) != (args.t2i_adapter_image is None):
        raise SystemExit("--t2i_adapter and --t2i_adapter_image go together")
    if (args.controlnet is None) != (args.control_image is None):
        raise SystemExit("--controlnet and --control_image go together")
    if (args.ip_adapter is None) != (args.ip_adapter_image is None):
        raise SystemExit("--ip_adapter and --ip_adapter_image go together")
    if args.denoising_end is not None and args.model != "sdxl":
        raise SystemExit("--denoising_end needs --model sdxl")

    set_seed(args.seed)
    create_workdir(args.workdir)
    solver_config = SimpleNamespace(num_sampling=args.NFE)  # the reference munchifies {'num_sampling': NFE}
    callback = None

    sdxl = args.model in ("sdxl", "sdxl_lightning")
    solver = build_solver(args.model, args.method, solver_config, args.device, args.ckpt_dir)
    for spec in args.lora:
        path, _, scale = spec.partition(":")
        solver.load_lora(path, float(scale) if scale else 1.0)
    native = solver.cfg.sample_size * 8
    height, width = args.height or native, args.width or native
    if height % 8 or width % 8:
        raise SystemExit(f"--height / --width must be multiples of 8 (got {height} x {width})")
    zT = draw_latents((1, 4, height // 8, width // 8))  # N(0, 1) start latent from the seeded CPU generator
    control = {}
    if args.controlnet is not None:
        from cfgpp_b200.controlnet import ControlNet
        control = {"controlnet": ControlNet(args.controlnet, args.device, base_cfg=solver.cfg),
                   "control_image": load_control_image(args.control_image, height, width),
                   "controlnet_conditioning_scale": args.controlnet_scale,
                   "control_guidance_start": args.control_guidance_start,
                   "control_guidance_end": args.control_guidance_end}
    if args.ip_adapter is not None:
        from PIL import Image
        from cfgpp_b200.ip_adapter import IPAdapter
        control.update(ip_adapter=IPAdapter(args.ip_adapter, args.device, solver.cfg,
                                            image_encoder=str(args.image_encoder) if args.image_encoder else None),
                       ip_adapter_image=Image.open(args.ip_adapter_image), ip_adapter_scale=args.ip_adapter_scale)
    if args.t2i_adapter is not None:
        from cfgpp_b200.t2i_adapter import T2IAdapter
        ad = T2IAdapter(args.t2i_adapter, args.device, base_cfg=solver.cfg)
        control.update(t2i_adapter=ad, adapter_conditioning_scale=args.adapter_conditioning_scale,
                       adapter_conditioning_factor=args.adapter_conditioning_factor,
                       t2i_adapter_image=load_control_image(args.t2i_adapter_image, height, width,
                                                            "L" if ad.cfg.in_channels == 1 else "RGB",
                                                            "--t2i_adapter_image"))
    if sdxl:
        refiner = {}
        if args.denoising_end is not None:
            refiner = {"refiner": build_refiner(args.device, args.refiner_ckpt_dir),
                       "denoising_end": args.denoising_end}
        result = solver.sample(prompt1=[args.null_prompt, args.prompt], prompt2=[args.null_prompt, args.prompt],
                               cfg_guidance=args.cfg_guidance, original_size=(height, width),
                               target_size=(height, width), callback_fn=callback, zT=zT, **refiner, **control)
    else:
        result = solver.sample(prompt=[args.null_prompt, args.prompt], cfg_guidance=args.cfg_guidance,
                               callback_fn=callback, zT=zT, **control)

    out = args.workdir.joinpath('result/generated.pt')
    torch.save(result, out)
    try:
        from torchvision.utils import save_image
        save_image(result, args.workdir.joinpath('result/generated.png'), normalize=True)
    except Exception:  # torchvision is optional here
        pass
    print(f"saved {out}")


def load_control_image(path: Path, height: int, width: int, mode: str = "RGB",
                       flag: str = "--control_image") -> torch.Tensor:
    """(1, 3, H, W) RGB (mode "RGB") or (1, 1, H, W) grayscale (mode "L") in [0, 1]. The image must already have the
    output size: it is not resized."""
    import numpy as np
    from PIL import Image
    img = Image.open(path).convert(mode)
    if img.size != (width, height):
        raise SystemExit(f"{flag} is {img.size[0]} x {img.size[1]}, the output is {width} x {height}")
    x = torch.from_numpy(np.asarray(img).copy())
    x = x[None] if x.dim() == 2 else x.permute(2, 0, 1)
    return x[None].float() / 255.0


if __name__ == "__main__":
    main()
