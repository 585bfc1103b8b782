"""Step time of the DINOv3 SAM encoder distillation (13.interactive_segmentation_training/13.0.encoder_distill_training,
sam_h_encoder_distill_dinov3_vit_base_patch16_encoder) at its per-GPU shape: 1024 x 1024 images, batch 16 (128 over 8
GPUs).  One step = SAM ViT-H teacher forward (no grad) + DINOv3 ViT-B/16 + neck student forward and backward + MSELoss +
FusedAdamW.  Timed with CUDA events after warm-up; the card's name and power limit are read in the same run.  --profile
adds a separate torch.profiler run that reports the share of the step spent in the RoPE, SwiGLU and layer-scale kernels
(the full kernel table goes to --out).
When the reference is installed (oracle/_ref), its model is timed under autocast(bf16) with torch.optim.AdamW at the same
shape on the same card.

    python tests/perf_dinov3_distill.py [--batch 16] [--size 1024] [--steps 10] [--warmup 3] [--profile] [--reference]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = f'{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})'
    return q


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(steps):
        step()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / steps


def runtime_step(batch, size):
    from simpleaicv_pytorch_training_examples_b200 import optim
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation import distill_model
    from simpleaicv_pytorch_training_examples_b200.interactive_segmentation.distill_losses import MSELoss
    torch.manual_seed(0)
    tea = dict(distill_model.SAM_H_TEACHER, image_size=size)
    stu = dict(distill_model.DINOV3_B_STUDENT, image_size=size)
    model = distill_model.DINOV3ImageEncoderDistillModel(teacher_params=tea, student_params=stu).cuda().train()
    model.teacher.eval()
    opt = optim.FusedAdamW([{'params': [p for p in model.parameters() if p.requires_grad], 'weight_decay': 0.}], lr=1e-5)
    crit = MSELoss()
    x = torch.randn(batch, 3, size, size, device='cuda')

    def step():
        tea_out, stu_out = model(x)
        crit(tea_out, stu_out)['distill_mse_loss'].backward()
        opt.step()
        opt.zero_grad()
    return step


def reference_step(batch, size):
    from baseline import ref_import
    dm = ref_import.module('SimpleAICV.interactive_segmentation.distill_model')
    dl = ref_import.module('SimpleAICV.interactive_segmentation.distill_losses')
    torch.manual_seed(0)
    model = dm.DINOV3ImageEncoderDistillModel(
        teacher_params={'image_size': size, 'patch_size': 16, 'inplanes': 3, 'embedding_planes': 1280, 'block_nums': 32, 'head_nums': 16,
                        'mlp_ratio': 4, 'out_planes': 256, 'window_size': 14, 'global_attn_indexes': [7, 15, 23, 31],
                        'use_gradient_checkpoint': False},
        student_params={'backbone_type': 'dinov3_vit_base_patch16_backbone', 'image_size': size, 'out_planes': 256,
                        'use_gradient_checkpoint': False}).cuda().train()
    model.teacher.eval()
    opt = torch.optim.AdamW([p for p in model.parameters() if p.requires_grad], lr=1e-5, weight_decay=0.)
    crit = dl.MSELoss()
    x = torch.randn(batch, 3, size, size, device='cuda')

    def step():
        with torch.autocast('cuda', dtype=torch.bfloat16):
            tea_out, stu_out = model(x)
            loss = crit(tea_out, stu_out)['distill_mse_loss']
        loss.backward()
        opt.step()
        opt.zero_grad()
    return step


def profile(step, out_dir):
    from torch.profiler import ProfilerActivity, profile as tprofile
    step()
    torch.cuda.synchronize()
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
            step()
        torch.cuda.synchronize()
    groups = {'rope': 0., 'swiglu': 0., 'ls_residual': 0., 'gemm': 0., 'attn': 0.}
    total = 0.
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, 'device_time_total') else e.cuda_time_total
        total += t
        for k in groups:
            if k in e.key:
                groups[k] += t
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, 'dinov3_distill_kernels.txt'), 'w') as f:
        f.write(prof.key_averages().table(sort_by='cuda_time_total', row_limit=40))
    return {k: {'ms_per_step': v / 2e3, 'share': v / total if total else 0.} for k, v in groups.items()}, total / 2e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=16)
    ap.add_argument('--size', type=int, default=1024)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--profile', action='store_true')
    ap.add_argument('--reference', action='store_true')
    ap.add_argument('--out', default=os.path.join(tempfile.gettempdir(), 'perf_dinov3_distill'),
                    help='directory for the --profile kernel table')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'this measurement needs the GPU'
    res = {'card': card(), 'batch': a.batch, 'size': a.size}
    step = runtime_step(a.batch, a.size)
    ms = time_steps(step, a.steps, a.warmup)
    res.update(step_ms=ms, img_per_s=a.batch * 1e3 / ms, peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
    if a.profile:
        res['kernels'], res['profiled_gpu_ms_per_step'] = profile(step, a.out)
    del step
    torch.cuda.empty_cache()
    if a.reference:
        from baseline import ref_import
        if ref_import.available():
            try:
                torch.cuda.reset_peak_memory_stats()
                rms = time_steps(reference_step(a.batch, a.size), a.steps, a.warmup)
                res.update(reference_step_ms=rms, reference_img_per_s=a.batch * 1e3 / rms,
                           reference_peak_mem_gb=torch.cuda.max_memory_allocated() / 2 ** 30)
            except torch.cuda.OutOfMemoryError:
                res['reference_step_ms'] = 'out of memory'
        else:
            res['reference_step_ms'] = 'reference not installed'
    print(json.dumps(res))


if __name__ == '__main__':
    main()
