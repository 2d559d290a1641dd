"""CLI with the reference's flag surface (examples/inversion.py:23-37): invert an image with the source prompt and
reconstruct / edit it —
    python -m examples.inversion --method ddim_inversion_cfg++ --NFE 10 --cfg_guidance 0.6 --prompt "a cat"
    python -m examples.inversion --method ddim_edit_cfg++ --prompt "a cat" --tgt_prompt "a dog"
Runs on the Hopper-native (sm_90a) backend (both loops are fused CUDA-graph trajectories). Offline the UNet weights are
seeded synthetic and the text encoder / VAE are stand-ins (cfgpp_b200/conditioning.py): a plumbing check."""
import argparse
from pathlib import Path
from types import SimpleNamespace

import torch

from cfgpp_b200.checkpoints import solver_components
from examples.text_to_img import build_solver
from cfgpp_b200.latent_diffusion import get_solver
from cfgpp_b200.latent_sdxl import get_solver as get_solver_sdxl
from cfgpp_b200.utils.log_util import create_workdir, set_seed


def load_img(img_path: Path, size: int = 512, centered: bool = True) -> torch.Tensor:
    """(1,3,size,size) in [-1,1]; a smooth synthetic image when the file or PIL is missing (offline image)."""
    try:
        import numpy as np
        from PIL import Image
        image = torch.from_numpy(np.array(Image.open(img_path).convert('RGB').resize((size, size)))).permute(2, 0, 1)
        image = image / 127.5 - 1 if centered else image
    except Exception:
        ys, xs = torch.meshgrid(torch.linspace(-1, 1, size), torch.linspace(-1, 1, size), indexing="ij")
        image = torch.stack([torch.sin(3 * xs) * torch.cos(2 * ys), xs * ys, torch.cos(4 * (xs + ys))])
    return image.unsqueeze(0).float()


def main():
    parser = argparse.ArgumentParser(description="Latent Diffusion")
    parser.add_argument("--workdir", type=Path, default="examples/workdir/inversion")
    parser.add_argument("--img_path", type=Path, default="examples/assets/afhq_1.jpg")
    parser.add_argument("--img_size", type=int, default=None,
                        help="square image size (default: the model's native size, 512 / 768 (sd20) / 1024)")
    parser.add_argument("--device", type=str, default="cuda")
    parser.add_argument("--null_prompt", type=str, default="")
    parser.add_argument("--prompt", type=str, default="")
    parser.add_argument("--tgt_prompt", type=str, default=None, help="target prompt of the *_edit* methods")
    parser.add_argument("--cfg_guidance", type=float, default=7.5)
    parser.add_argument("--method", type=str, default='ddim_inversion_cfg++')
    parser.add_argument("--model", type=str, default='sd15', choices=["sd15", "sd20", "sdxl"])
    parser.add_argument("--NFE", type=int, default=10)
    parser.add_argument("--seed", type=int, default=42)
    parser.add_argument("--ckpt_dir", type=Path, default=None,
                        help="diffusers-format pipeline directory (unet/, vae/, text_encoder[_2]/, tokenizer[_2]/); "
                             "default: seeded synthetic weights (nothing can be downloaded here)")
    args = parser.parse_args()

    set_seed(args.seed)
    create_workdir(args.workdir)
    solver_config = SimpleNamespace(num_sampling=args.NFE)
    if args.img_size is None:
        args.img_size = {"sd15": 512, "sd20": 768, "sdxl": 1024}[args.model]
    img = load_img(args.img_path, size=args.img_size)
    prompts = [args.null_prompt, args.prompt, args.tgt_prompt if args.tgt_prompt is not None else args.prompt]

    if args.model == "sdxl":
        extra = solver_components(args.ckpt_dir, "sdxl", args.device) if args.ckpt_dir else {}
        solver = get_solver_sdxl(args.method, solver_config=solver_config, device=args.device, **extra)
        result = solver.sample(prompt1=prompts, prompt2=prompts, src_img=img, cfg_guidance=args.cfg_guidance,
                               target_size=(args.img_size, args.img_size))
    else:
        solver = build_solver(args.model, args.method, solver_config, args.device, args.ckpt_dir)
        result = solver.sample(prompt=prompts, src_img=img, cfg_guidance=args.cfg_guidance, callback_fn=None)

    out = args.workdir.joinpath('result/reconstruct.pt')
    torch.save(result, out)
    try:
        from torchvision.utils import save_image
        save_image(result, args.workdir.joinpath('result/reconstruct.png'), normalize=True)
    except Exception:  # torchvision is optional here
        pass
    print(f"saved {out}")


if __name__ == "__main__":
    main()
