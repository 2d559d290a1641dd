"""Many-prompt generation with the reference's flag surface (examples/text_to_mscoco.py:14-26) —
    python -m examples.text_to_mscoco --model sdxl --method ddim_cfg++ --cfg_guidance 0.6 --prompt_dir prompts.txt
    torchrun --nproc-per-node 8 --master-addr 127.0.0.1 -m examples.text_to_mscoco --model sdxl ...
The reference loops over the prompts on one GPU. Here prompt i goes to rank i % world (SURVEY section 8e): every rank
holds a full UNet replica, rank 0's weights are broadcast once over NCCL so the replicas are bit-identical, and there
is no collective inside the sampling loop. Every rank draws the zT of EVERY image from the seeded CPU generator, in
order, and keeps its own - so image i is the same picture whatever the world size. `--batch_size B` groups each rank's
prompts into batches of up to B images that share one trajectory (UNet batch 2B, B <= 8); the zT draws stay per image,
so image i does not depend on B either (its pixels may differ in the last bits: other GEMM shapes)."""
import argparse
import os
from pathlib import Path
from types import SimpleNamespace

import torch

from cfgpp_b200 import dist as D
from cfgpp_b200 import weights as Wt
from cfgpp_b200.config import sd2_config, sd15_config, sdxl_config
from cfgpp_b200.latent_diffusion import get_solver
from cfgpp_b200.latent_sdxl import get_solver as get_solver_sdxl
from cfgpp_b200.utils.log_util import create_workdir, set_seed
from examples.text_to_img import model_family


def read_prompts(path: Path, limit: int = 10000):
    if not Path(path).exists():
        return [f"synthetic prompt {i}" for i in range(8)]  # offline: no MS-COCO caption file
    with open(path, 'r') as f:
        return [ln.strip() for ln in f if ln.strip()][:limit]


def rank_batches(n_prompts: int, rank: int, world: int, batch_size: int, latent):
    """Yield (image indices, zT) for this rank: its prompts (i % world == rank) in order, grouped by `batch_size`.
    zT is drawn from the CPU generator for every image 0..n-1 in order on every rank, and each rank keeps the draws
    of its own images."""
    if batch_size < 1:
        raise ValueError("--batch_size must be >= 1")
    mine = set(D.shard_indices(n_prompts, rank, world))
    idx, zs = [], []
    for i in range(n_prompts):
        zT = torch.randn(latent)  # CPU generator, advanced for every image on every rank (see module docstring)
        if i not in mine:
            continue
        idx.append(i)
        zs.append(zT)
        if len(idx) == batch_size:
            yield idx, torch.cat(zs)
            idx, zs = [], []
    if idx:
        yield idx, torch.cat(zs)


def main():
    parser = argparse.ArgumentParser(description="Latent Diffusion")
    parser.add_argument("--workdir", type=Path, default="examples/workdir/mscoco")
    parser.add_argument('--prompt_dir', type=Path, default=Path('examples/assets/coco_v2.txt'))
    parser.add_argument("--device", type=str, default="cuda")
    parser.add_argument("--null_prompt", type=str, default="")
    parser.add_argument("--prompt", type=str, default="")
    parser.add_argument("--cfg_guidance", type=float, default=7.5)
    parser.add_argument("--method", type=str, default='ddim')
    parser.add_argument("--model", type=str, default='sd15', choices=["sd15", "sd20", "sdxl", "sdxl_lightning"])
    parser.add_argument("--NFE", type=int, default=50)
    parser.add_argument("--seed", type=int, default=42)
    parser.add_argument("--batch_size", type=int, default=1,
                        help="images per trajectory (1..8); every image keeps its own zT and result file")
    parser.add_argument("--ckpt_dir", type=Path, default=None,
                        help="diffusers-format pipeline directory (unet/, vae/, text_encoder[_2]/, tokenizer[_2]/); "
                             "default: seeded synthetic weights (nothing can be downloaded here)")
    args = parser.parse_args()

    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    device = torch.device("cuda", local) if world > 1 else torch.device(args.device)
    if world > 1:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=device)

    set_seed(args.seed)
    if rank == 0:
        create_workdir(args.workdir)
    text_list = read_prompts(args.prompt_dir)
    solver_config = SimpleNamespace(num_sampling=args.NFE)
    family = model_family(args.model)
    sdxl = family == "sdxl"
    cfg = {"sd15": sd15_config, "sd20": sd2_config, "sdxl": sdxl_config}[family]()

    kw = {} if sdxl else {"unet_config": cfg}
    if args.ckpt_dir:  # every rank reads the pipeline directory itself (UNet, VAE, text towers, tokenizers)
        from cfgpp_b200.checkpoints import solver_components
        kw.update(solver_components(args.ckpt_dir, family, device))
        cfg = kw.get("unet_config", cfg)
    elif world > 1:  # one bucketed NCCL broadcast of rank 0's weights; afterwards the ranks never talk again
        sd = Wt.synthetic_state_dict(cfg, seed=1234, device=device) if rank == 0 else None
        kw["state_dict"] = D.broadcast_state_dict(sd, Wt.unet_param_specs(cfg), device, src=0)
    solver = (get_solver_sdxl if sdxl else get_solver)(args.method, solver_config=solver_config, device=device, **kw)

    latent = (1, 4, cfg.sample_size, cfg.sample_size)
    for idx, zT in rank_batches(len(text_list), rank, world, args.batch_size, latent):
        texts = [text_list[i] for i in idx]
        for i, text in zip(idx, texts):
            print(f'[rank {rank}] processing {i + 1}/{len(text_list)}: {text}', flush=True)
        if sdxl:
            results = solver.sample(prompt1=[args.null_prompt, texts], prompt2=[args.null_prompt, texts],
                                    cfg_guidance=args.cfg_guidance, target_size=(1024, 1024), zT=zT)
        else:
            results = solver.sample(prompt=[args.null_prompt, texts], cfg_guidance=args.cfg_guidance, zT=zT)
        for j, i in enumerate(idx):
            result = results[j:j + 1]
            torch.save(result, args.workdir.joinpath(f'{str(i).zfill(5)}.pt'))
            try:
                from torchvision.utils import save_image
                save_image(result, args.workdir.joinpath(f'{str(i).zfill(5)}.png'), normalize=True)
            except Exception:  # torchvision is optional here
                pass
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
