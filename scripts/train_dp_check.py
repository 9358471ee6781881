"""Data-parallel codebook training step: N ranks x (B/N) images must reproduce 1 rank x B images (gradient average over NCCL,
packed EMA-statistics all-reduce).  Run under torchrun (NCCL); rank 0 also runs the full batch alone and compares.
Also times a full-size step (config 4 shape: 32 images per GPU)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from oracle import synth
from oracle.make_golden import SMALL_VQ, vq_images
from viewformer_b200 import VQGAN
from viewformer_b200.config import VQGANConfig
from viewformer_b200.train import VQGANTrainer

world, rank, local = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
if world > 1:
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
cfg = VQGANConfig(**dict(SMALL_VQ, perceptual_weight=0.0))
sd = synth.make_vqgan_state_dict(cfg, 5)
B = 4 * world
x = vq_images(B, cfg.image_size, 123)
tr = VQGANTrainer(VQGAN(cfg, precision="fp32", device=f"cuda:{local}").load_state_dict(sd), bucket_bytes=1 << 18)
loss = tr.forward_backward(x[rank * 4:(rank + 1) * 4])
tr.ex.wait()
g_dp = tr.flat_g.clone() / world                 # the optimizer applies the same 1 / world (DDP gradient average)
tr.optimizer_step()
torch.cuda.synchronize()
mine = tr.export_state_dict()
if world > 1:
    lt = torch.tensor([float(loss)], device=f"cuda:{local}")
    dist.all_reduce(lt)
    lmean = float(lt) / world
    dist.barrier()
else:
    lmean = float(loss)
if world > 1:
    # reference run: the WHOLE batch on one GPU.  Every rank builds a 1-member group (new_group is collective) and repeats the step
    # alone, with the EMA-statistics exchange switched off
    groups = [dist.new_group([r]) for r in range(world)]
    solo_group = groups[rank]
    tr1 = VQGANTrainer(VQGAN(cfg, precision="fp32", device=f"cuda:{local}").load_state_dict(sd), bucket_bytes=1 << 18, process_group=solo_group)
    from viewformer_b200 import dist as vdist
    _orig = vdist.allreduce_ema_stats
    vdist.allreduce_ema_stats = lambda c, e, group=None: (c, e)          # the solo run must not exchange EMA statistics
    l1 = tr1.forward_backward(x)
    g_full = tr1.flat_g.clone()
    tr1.optimizer_step()
    vdist.allreduce_ema_stats = _orig
    torch.cuda.synchronize()
    solo = tr1.export_state_dict()
    if rank == 0:
        worst = max(float((mine[k].float() - solo[k].float()).abs().max()) for k in solo if solo[k].dtype.is_floating_point)
        grel = float((g_dp - g_full).norm() / g_full.norm())
        print(f"[dp check] world {world}: mean loss over ranks {lmean:.6f} vs single-GPU full batch {float(l1):.6f}; "
              f"gradient |g_dp - g_full| / |g_full| = {grel:.2e}; max |weight difference| after one Adam step {worst:.3e} (lr {cfg.learning_rate}; "
              f"Adam's first step moves every weight by ~lr * sign(g), so elements whose true gradient is zero differ by up to lr)")
    dist.barrier()
# ---- full-size step timing (BASELINE config 4 shape: 32 images per GPU, fp32)
fcfg = VQGANConfig(perceptual_weight=0.0)
n_img = int(os.environ.get("VF_TRAIN_IMAGES", "32"))
trf = VQGANTrainer(VQGAN(fcfg, precision="fp32", device=f"cuda:{local}").init_weights(0))
xf = torch.rand((n_img, 3, 128, 128), generator=torch.Generator().manual_seed(rank)) * 2 - 1
trf.training_step(xf)
torch.cuda.synchronize()
if world > 1:
    dist.barrier()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
steps = 2
for _ in range(steps):
    lossf = trf.training_step(xf)
e1.record()
torch.cuda.synchronize()
ms = torch.tensor([e0.elapsed_time(e1) / steps], device=f"cuda:{local}")
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
if rank == 0:
    print(f"[train step, full size] {world} GPU(s) x {n_img} images: {float(ms):.1f} ms/step -> {world * n_img / float(ms) * 1e3:.1f} images/s; "
          f"loss {float(lossf):.4f}; {len(trf.buckets)} gradient buckets of <= {trf.bucket_bytes >> 20} MiB over {trf.flat_g.numel() * 4 >> 20} MiB")
if world > 1:
    dist.destroy_process_group()
