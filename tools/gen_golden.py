#!/usr/bin/env python
"""Generate tests/golden/* by importing the UNMODIFIED reference (a read-only checkout named by DPB200_REFERENCE).

Needs the reference checkout and CPUs only:
    DPB200_REFERENCE=<checkout> python tools/gen_golden.py [--skip-cfg1] [--only NAME]
Outputs (all small, committed):
    tests/golden/tiny_unet.pt      TINY config: inputs, output, loss, all grads after 1 pass (B=2)
    tests/golden/blocks.pt         one ResnetBlock2D (with shortcut) and one Attention: in/out/grads
    tests/golden/cifar_fwd.pt      C1 seed-0: state-dict fingerprints, eps_hat for B=2 at t in {0,500,999},
                                   KAT losses at B=16 t in {0,50,99}, grad fingerprints after one pass
    tests/golden/cifar_cfg1.pt     BASELINE config 1 (B=16, t=0..99, ratio 0.3): per importance variant, the
                                   interactive group sequence (structure, importance vector, pruned indices),
                                   post-prune shapes / param+MAC counts / pruned-model eps
    tests/golden/cifar_cfg1_s3.pt  same with 3 timesteps (fast CPU check of the oracle)
    tests/golden/finetune_tiny.pt  2 finetune steps on TINY (Adam + clip + EMA), dropout 0
    tests/golden/ddim_tiny.pt      DDIMPipeline samples (uniform/eta 0/10 steps, quad/eta 0.5/7 steps) on TINY
    tests/golden/fid_*             FID Inception fixtures (gen_fid): weight-file layout, features of seeded weights, Frechet cases
    tests/golden/ssim_ref.pt       SSIM fixtures (gen_ssim): uint8 image pairs and utils_image.py's per-channel / per-image SSIM
    tests/golden/vq_decoder_tiny.pt  the LDM's VQ first-stage Decoder (small config and VQ-f4 at a 16 x 16 latent) and nearest-code choices
    tests/golden/vq_encoder_tiny.pt  the LDM's VQ first-stage Encoder and VQModelInterface.encode (small config and VQ-f4 at 64 x 64)
    tests/golden/ldm_ddim_tiny.pt  guided DDIM sampling of the tiny LDM by ldm_exp's DDIMSampler, every step, and one get_loss_at_t pass
"""
import argparse
import hashlib
import json
import os
import sys
import time

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import ref_shim  # noqa: E402

diffusers, tp = ref_shim.install()
from diffusers import DDPMScheduler, UNet2DModel  # noqa: E402
from diffusers.models.attention_processor import Attention, AttnProcessor  # noqa: E402
from diffusers.models.resnet import Downsample2D, ResnetBlock2D, Upsample2D  # noqa: E402
from torch_pruning.pruner import function as tpf  # noqa: E402

import diff_pruning_b200 as dp  # noqa: E402  (configs only)

OUT = os.path.join(ROOT, "tests", "golden")
os.makedirs(OUT, exist_ok=True)


def legacy_attn(model):
    for m in model.modules():
        if isinstance(m, Attention):
            m.set_processor(AttnProcessor())


def fp(t):
    t = t.detach().double()
    return [float(t.sum()), float(t.abs().sum()), float((t * t).sum())]


def build(cfg, seed=0):
    torch.manual_seed(seed)
    m = UNet2DModel(**cfg).eval()
    legacy_attn(m)  # identical math to 2_0 pre-pruning, and the only one that survives pruning
    return m


def inputs(b, hw, c=3):
    g1, g2 = torch.Generator().manual_seed(1), torch.Generator().manual_seed(2)
    return torch.randn(b, c, hw, hw, generator=g1), torch.randn(b, c, hw, hw, generator=g2)


def gen_tiny():
    cfg = dict(dp.TINY_TEST_CONFIG)
    m = build(cfg)
    sched = DDPMScheduler(num_train_timesteps=1000)
    clean, noise = inputs(2, 16)
    t = torch.tensor([7, 7]).long()
    m.zero_grad()
    losses = []
    for tt in (7, 400):  # two accumulated passes (no zero_grad in between)
        t = (tt * torch.ones(2)).long()
        out = m(sched.add_noise(clean, noise, t), t).sample
        loss = torch.nn.functional.mse_loss(out, noise)
        loss.backward()
        losses.append(loss.item())
    with torch.no_grad():
        t2 = torch.tensor([3, 950]).long()  # per-sample timesteps (finetune style)
        out2 = m(sched.add_noise(clean, noise, t2), t2).sample
    torch.save({"cfg": cfg, "seed": 0, "losses": losses, "out_last": out.detach(), "t2": t2, "out_t2": out2,
                "grads": {k: p.grad.clone() for k, p in m.named_parameters()}},
               os.path.join(OUT, "tiny_unet.pt"))
    print("tiny", losses)


def gen_blocks():
    torch.manual_seed(3)
    rb = ResnetBlock2D(in_channels=32, out_channels=64, temb_channels=128, groups=8, eps=1e-6)
    x = torch.randn(2, 32, 8, 8, requires_grad=True)
    temb = torch.randn(2, 128, requires_grad=True)
    y = rb(x, temb)
    gy = torch.randn_like(y)
    y.backward(gy)
    res = {"sd": {k: v.clone() for k, v in rb.state_dict().items()}, "x": x.detach(), "temb": temb.detach(),
           "y": y.detach(), "gy": gy, "gx": x.grad.clone(), "gtemb": temb.grad.clone(),
           "grads": {k: p.grad.clone() for k, p in rb.named_parameters()}}
    torch.manual_seed(4)
    at = Attention(64, heads=1, dim_head=64, rescale_output_factor=1.0, eps=1e-6, norm_num_groups=8,
                   residual_connection=True, bias=True, upcast_softmax=True, _from_deprecated_attn_block=True)
    at.set_processor(AttnProcessor())
    xa = torch.randn(2, 64, 4, 4, requires_grad=True)
    ya = at(xa)
    gya = torch.randn_like(ya)
    ya.backward(gya)
    att = {"sd": {k: v.clone() for k, v in at.state_dict().items()}, "x": xa.detach(), "y": ya.detach(), "gy": gya,
           "gx": xa.grad.clone(), "grads": {k: p.grad.clone() for k, p in at.named_parameters()}, "scale": at.scale}
    torch.save({"resnet": res, "attn": att}, os.path.join(OUT, "blocks.pt"))
    print("blocks ok")


def cifar_cfg():
    cfg = json.load(open(os.path.join(ref_shim.REF, "tools", "ddpm_cifar10_config.json")))
    return {k: v for k, v in cfg.items() if not k.startswith("_")}


def gen_cifar_fwd():
    m = build(cifar_cfg())
    sched = DDPMScheduler(num_train_timesteps=1000)
    sd = m.state_dict()
    res = {"sd_fp": {k: fp(v) for k, v in sd.items()},
           "sd_sha": hashlib.sha256(b"".join(v.numpy().tobytes() for v in sd.values())).hexdigest(),
           "n_params": sum(p.numel() for p in m.parameters())}
    clean16, noise16 = inputs(16, 32)
    kat = {}
    with torch.no_grad():
        for tt in (0, 50, 99):
            t = (tt * torch.ones(16)).long()
            out = m(sched.add_noise(clean16, noise16, t), t).sample
            kat[tt] = torch.nn.functional.mse_loss(out, noise16).item()
    res["kat_losses_b16"] = kat
    clean, noise = clean16[:2].clone(), noise16[:2].clone()
    eps = {}
    with torch.no_grad():
        for tt in (0, 500, 999):
            t = (tt * torch.ones(2)).long()
            eps[tt] = m(sched.add_noise(clean, noise, t), t).sample.clone()
    res["eps_b2"] = eps
    m.zero_grad()
    t = (500 * torch.ones(2)).long()
    out = m(sched.add_noise(clean, noise, t), t).sample
    loss = torch.nn.functional.mse_loss(out, noise)
    loss.backward()
    res["loss_b2_t500"] = loss.item()
    res["grad_fp_b2_t500"] = {k: fp(p.grad) for k, p in m.named_parameters()}
    res["grad_samples_b2_t500"] = {k: p.grad.flatten()[:64].clone() for k, p in m.named_parameters()}
    torch.save(res, os.path.join(OUT, "cifar_fwd.pt"))
    print("cifar_fwd", kat, res["loss_b2_t500"])


KIND = {tpf.prune_conv_out_channels: "out", tpf.prune_linear_out_channels: "out",
        tpf.prune_conv_in_channels: "in", tpf.prune_linear_in_channels: "in",
        tpf.prune_groupnorm_out_channels: "gn"}


def describe_group(group, names):
    items = []
    for dep, idxs in group:
        layer = dep.target.module
        kind = KIND.get(dep.handler)
        if layer not in names or kind is None:
            continue  # non-parametric nodes (concat/split/elementwise) carry no score
        if kind == "gn" and not layer.affine:
            continue
        items.append((names[layer], kind, [int(i) for i in idxs]))
    return items


def compress(idxs):
    idxs = [int(i) for i in idxs]
    if idxs and idxs == list(range(idxs[0], idxs[0] + len(idxs))):
        return ("range", idxs[0], len(idxs))
    return idxs


def describe_group_c(group, names):
    return [(n, k, compress(i)) for n, k, i in describe_group(group, names)]


class VariantTaylor:
    """reference importance.py:375-434 with :393/:407 switched per variant (SURVEY.md §8(c)); :416 for GroupNorm."""

    def __init__(self, variant):
        self.variant = variant

    @torch.no_grad()
    def __call__(self, group, ch_groups=1):
        imps = []
        for dep, idxs in group:
            idxs.sort()
            layer, fn = dep.target.module, dep.handler
            if fn in (tpf.prune_conv_out_channels, tpf.prune_linear_out_channels):
                w, dw = layer.weight.data[idxs].flatten(1), layer.weight.grad.data[idxs].flatten(1)
            elif fn in (tpf.prune_conv_in_channels, tpf.prune_linear_in_channels):
                w = layer.weight.data.transpose(0, 1).flatten(1)[idxs]
                dw = layer.weight.grad.data.transpose(0, 1).flatten(1)[idxs]
            elif fn == tpf.prune_groupnorm_out_channels:
                if layer.affine:
                    imps.append((layer.weight.data[idxs] * layer.weight.grad.data[idxs]).abs())
                continue
            else:
                continue
            p = w * dw
            imps.append({"vendored": p.abs().pow(2).sum(1), "taylor": p.sum(1).abs(), "diff": p.abs().sum(1)}[self.variant])
        if not imps:
            return None
        size = len(imps[0])
        return torch.stack([i for i in imps if len(i) == size], 0).sum(0)


def gen_cfg1(n_steps=100, ratio=0.3, B=16, out_name="cifar_cfg1.pt", cfg=None, hw=32, timesteps=None, eps_stride=None):
    import copy
    os.chdir("/tmp")  # prune_local writes ./run/pruning_logs
    m0 = build(cifar_cfg() if cfg is None else cfg)
    sched = DDPMScheduler(num_train_timesteps=1000)
    clean, noise = inputs(B, hw)
    example = {"sample": torch.randn(1, 3, hw, hw), "timestep": torch.ones((1,)).long()}
    m0.zero_grad()
    m0.eval()
    losses, eps_sub = [], []
    t0 = time.time()
    timesteps = list(range(n_steps)) if timesteps is None else list(timesteps)
    cache = os.path.join("/tmp", out_name + ".passes")          # scratch cache of the (slow) passes while iterating on this script
    if os.path.exists(cache):
        c = torch.load(cache, weights_only=False)
        losses, eps_sub = c["losses"], c["eps_sub"]
        for k_, p_ in m0.named_parameters():
            p_.grad = c["grads"][k_]
        timesteps_run = []
    else:
        timesteps_run = timesteps
    for k in timesteps_run:
        t = (k * torch.ones(B)).long()
        out = m0(sched.add_noise(clean, noise, t), t).sample
        loss = torch.nn.functional.mse_loss(out, noise)
        loss.backward()
        losses.append(loss.item())
        if eps_stride:   # strided sample of eps_hat (the full tensor would be MBs per timestep)
            eps_sub.append(out.detach()[:, :, ::eps_stride, ::eps_stride].clone())
        if k % 10 == 0 or hw > 32:
            print(f"  {out_name} pass t={k} loss {losses[-1]:.7f} ({time.time() - t0:.0f}s)", flush=True)
    if hw > 32 and not os.path.exists(cache):
        torch.save({"losses": losses, "eps_sub": eps_sub, "grads": {k_: p_.grad for k_, p_ in m0.named_parameters()}}, cache)
    grad_fp = {k: fp(p.grad) for k, p in m0.named_parameters()}
    res = {"n_steps": len(timesteps), "timesteps": timesteps, "ratio": ratio, "B": B, "hw": hw, "losses": losses, "grad_fp": grad_fp,
           "variants": {}}
    if eps_stride:
        res["eps_stride"], res["eps_sub"] = eps_stride, eps_sub
    for variant in ("vendored", "taylor", "diff"):
        m = copy.deepcopy(m0)
        for (k, p), (_, q) in zip(m.named_parameters(), m0.named_parameters()):
            p.grad = q.grad.clone()
        legacy_attn(m)
        names = {mod: n for n, mod in m.named_modules()}
        # the pinned behaviour: the vendored TaylorImportance class for "vendored" (unmodified reference code),
        # the same class body with the product/abs placement switched for the two pip forms.
        imp = tp.importance.TaylorImportance() if variant == "vendored" else VariantTaylor(variant)
        pruner = tp.pruner.MagnitudePruner(m, example, importance=imp, iterative_steps=1, channel_groups={},
                                           ch_sparsity=ratio, ignored_layers=[m.conv_out])
        base_macs, base_params = tp.utils.count_ops_and_params(m, example)
        checker = VariantTaylor(variant)
        groups = []
        # Scores are evaluated INTERACTIVELY: later groups see layers already sliced by earlier groups
        # (ddpm_prune.py:108-109 + metapruner.py:205-254), so record each group right before it is pruned.
        for g in pruner.step(interactive=True):
            module, fn = g[0][0].target.module, g[0][0].handler
            cur = pruner.DG.get_out_channels(module)
            full = pruner.DG.get_pruning_group(module, fn, list(range(cur)))
            ch_groups = pruner.get_channel_groups(full)
            sc = checker(full, ch_groups=ch_groups)
            sc_ref = imp(full, ch_groups=ch_groups)
            assert torch.equal(sc, sc_ref), names[module]
            sel = [int(i) for i in g[0][1]]
            full_items = describe_group(full, names)
            pr_items = describe_group(g, names)
            # index mapping is positional: pruned idxs of every item == its full idxs at the selected positions
            # (same traversal => same item order; a layer may appear twice when both halves of a concat are in the group)
            # (a GroupNorm-coupled group whose per-GN-group quota n_pruned // 32 is 0 — every such group at ratio 0.05 — is yielded
            #  with an EMPTY selection and prunes nothing: metapruner.py:237-246)
            assert len(full_items) == len(pr_items) or not sel
            for (n, k, i), (n2, k2, fi) in zip(pr_items if sel else [], full_items):
                # a layer fed by BOTH halves of a concat owned by this group appears once with the two index lists
                # merged (len = parts * channels); such items are skipped by the importance (:422-426) but pruned.
                parts = len(fi) // cur
                assert (n, k) == (n2, k2) and len(fi) == parts * cur, (n, k)
                assert sorted(i) == sorted(fi[q * cur + j] for q in range(parts) for j in sel), (n, k)
            n_pruned = cur - int(pruner.layer_init_out_ch[module] * (1 - pruner.get_target_sparsity(module)))
            groups.append({"root": names[module], "root_kind": KIND[fn], "ch_groups": int(ch_groups), "channels": int(cur),
                           "n_pruned": int(n_pruned), "items": [(n, k, compress(i)) for n, k, i in full_items],
                           "imp": sc.clone(), "idxs": sel})
            g.prune()
        for mod in m.modules():
            if isinstance(mod, (Upsample2D, Downsample2D)):
                mod.channels = mod.conv.in_channels
        macs, params = tp.utils.count_ops_and_params(m, example)
        shapes = {k: list(v.shape) for k, v in m.state_dict().items()}
        with torch.no_grad():  # pruned-model forward (legacy attention, stale scale)
            t = (10 * torch.ones(2)).long()
            out = m(sched.add_noise(clean[:2], noise[:2], t), t).sample
        res["variants"][variant] = {"groups": groups, "base": [base_macs, base_params], "pruned": [macs, params],
                                    "pruned_shapes": shapes,
                                    "pruned_eps_b2_t10": (out[:, :, ::eps_stride, ::eps_stride] if eps_stride else out).clone()}
        print("cfg1", variant, base_params, params, macs, len(groups), sum(len(g["idxs"]) for g in groups), flush=True)
    torch.save(res, os.path.join(OUT, out_name))


def gen_cfg1_s3():
    gen_cfg1(n_steps=3, out_name="cifar_cfg1_s3.pt")


def gen_cfg3_s3():
    """BASELINE config 3 (google/ddpm-ema-bedroom-256 architecture, README.md:140-148: --batch_size 4 --pruning_ratio 0.05) with 3 of
    the 1000 timesteps (t = 0, 500, 999): losses, a strided sample of eps_hat, gradient fingerprints and the interactive prune
    sequence (scores + selected channels) for all three importance variants.  ~2 CPU-minutes for the passes."""
    gen_cfg1(ratio=0.05, B=4, out_name="lsun_cfg3_s3.pt", cfg=dict(dp.LSUN256_DDPM_CONFIG), hw=256, timesteps=(0, 500, 999),
             eps_stride=4)


def gen_finetune():
    cfg = dict(dp.TINY_TEST_CONFIG)
    m = build(cfg).train()
    sched = DDPMScheduler(num_train_timesteps=1000)
    opt = torch.optim.Adam(m.parameters(), lr=2e-4, betas=(0.9, 0.999), weight_decay=0.0, eps=1e-8)
    from diffusers.training_utils import EMAModel
    ema = EMAModel(m.parameters(), decay=0.9999, use_ema_warmup=True, inv_gamma=1.0, power=0.75,
                   model_cls=UNet2DModel, model_config=m.config)
    g = torch.Generator().manual_seed(5)
    rec = {"cfg": cfg, "steps": []}
    for step in range(2):
        clean = torch.randn(4, 3, 16, 16, generator=g)
        noise = torch.randn(4, 3, 16, 16, generator=g)
        t = torch.randint(0, 1000, (4 // 2 + 1,), generator=g)
        t = torch.cat([t, 1000 - t - 1], dim=0)[:4]
        noisy = sched.add_noise(clean, noise, t)
        opt.zero_grad()
        out = m(noisy, t).sample
        loss = (noise - out).square().sum(dim=(1, 2, 3)).mean(dim=0)
        loss.backward()
        gn = torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        opt.step()
        ema.step(m.parameters())
        rec["steps"].append({"clean": clean, "noise": noise, "t": t, "loss": loss.item(), "grad_norm": gn.item()})
    rec["params"] = {k: p.detach().clone() for k, p in m.named_parameters()}
    rec["ema"] = {k: s.clone() for (k, _), s in zip(m.named_parameters(), ema.shadow_params)}
    torch.save(rec, os.path.join(OUT, "finetune_tiny.pt"))
    print("finetune", [s["loss"] for s in rec["steps"]], [s["grad_norm"] for s in rec["steps"]])


def gen_ddim():
    """DDIMPipeline (pipeline_ddim.py:45-122) + the reference's modified DDIMScheduler on the TINY UNet, CPU generator."""
    from diffusers import DDIMPipeline
    cfg = dict(dp.TINY_TEST_CONFIG)
    m = build(cfg)
    res = {"cfg": cfg}
    for name, skip, eta, steps in (("uniform_eta0", "uniform", 0.0, 10), ("quad_eta05", "quad", 0.5, 7)):
        pipe = DDIMPipeline(unet=m, scheduler=DDPMScheduler(num_train_timesteps=1000))
        pipe.scheduler.skip_type = skip
        pipe.set_progress_bar_config(disable=True)
        g = torch.Generator().manual_seed(0)
        out = pipe(batch_size=2, generator=g, eta=eta, num_inference_steps=steps, output_type="numpy").images
        res[name] = {"skip_type": skip, "eta": eta, "steps": steps, "images": torch.from_numpy(out),
                     "timesteps": pipe.scheduler.timesteps.clone()}
    torch.save(res, os.path.join(OUT, "ddim_tiny.pt"))
    print("ddim", {k: float(v["images"].mean()) for k, v in res.items() if k != "cfg"})


def gen_ckpt():
    """`DDPMPipeline.save_pretrained` of the reference's vendored diffusers (pipeline_utils.py:485-560, modeling_utils.py:250-330,
    configuration_utils.py:138-170) on the TINY UNet: keeps the three JSON files (the weights are the seeded tiny UNet, whose
    state-dict keys/shapes are pinned elsewhere) as tests/golden/ckpt_tiny_ref/, plus a digest of the state-dict it wrote."""
    import hashlib
    import shutil
    import tempfile
    from diffusers import DDPMPipeline
    m = build(dict(dp.TINY_TEST_CONFIG))
    pipe = DDPMPipeline(unet=m, scheduler=DDPMScheduler(num_train_timesteps=1000))
    tmp = tempfile.mkdtemp()
    pipe.save_pretrained(tmp)
    dst = os.path.join(OUT, "ckpt_tiny_ref")
    for rel in ("model_index.json", "unet/config.json", "scheduler/scheduler_config.json"):
        os.makedirs(os.path.dirname(os.path.join(dst, rel)), exist_ok=True)
        shutil.copy(os.path.join(tmp, rel), os.path.join(dst, rel))
    sd = torch.load(os.path.join(tmp, "unet", "diffusion_pytorch_model.bin"), map_location="cpu")
    h = hashlib.sha256()
    for k, v in sd.items():
        h.update(k.encode()); h.update(v.contiguous().numpy().tobytes())
    json.dump({"files": sorted(os.listdir(os.path.join(tmp, "unet"))), "n_tensors": len(sd), "state_dict_sha256": h.hexdigest()},
              open(os.path.join(dst, "weights_digest.json"), "w"), indent=1)
    shutil.rmtree(tmp)
    print("ckpt", len(sd), h.hexdigest()[:16])


def gen_lr():
    """diffusers.optimization.get_scheduler (optimization.py:282-340) sampled at a few optimiser steps: multipliers of the base lr."""
    from diffusers.optimization import get_scheduler
    out = {}
    for name in ("constant", "constant_with_warmup", "linear", "cosine"):
        for warm, total in ((0, 100), (5, 100), (500, 10000)):
            steps = sorted({0, 1, 2, warm - 1, warm, warm + 1, total // 2, total - 1, total, total + 3} - {-1})
            prm = torch.nn.Parameter(torch.zeros(1))
            opt = torch.optim.SGD([prm], lr=1.0)
            sch = get_scheduler(name, opt, num_warmup_steps=warm, num_training_steps=total)
            vals, k = {}, 0
            for s in range(max(steps) + 1):
                if s in steps:
                    vals[str(s)] = sch.get_last_lr()[0]
                opt.step(); sch.step()
            out[f"{name}|{warm}|{total}"] = vals
    json.dump(out, open(os.path.join(OUT, "lr_schedules.json"), "w"), indent=1)
    print("lr", len(out))


def gen_lsun_struct(ratio=0.05):
    """The six-level LSUN-256 architecture (google/ddpm-ema-bedroom-256: BASELINE config 3, ratio 0.05) at reduced widths
    (32, 32, 64, 64, 128, 128), `--pruner magnitude` (ddpm_prune.py:70-71: tp.importance.MagnitudeImportance()) through the
    interactive prune sequence: pins the structural group derivation, ch_groups, the per-group magnitude scores and the selected
    channel indices for the second headline architecture.  No gradients needed."""
    cfg = dict(dp.LSUN256_DDPM_CONFIG, block_out_channels=(32, 32, 64, 64, 128, 128))
    m = build(cfg)
    example = {"sample": torch.randn(1, 3, 64, 64), "timestep": torch.ones((1,)).long()}
    names = {mod: n for n, mod in m.named_modules()}
    imp = tp.importance.MagnitudeImportance()
    pruner = tp.pruner.MagnitudePruner(m, example, importance=imp, iterative_steps=1, channel_groups={}, ch_sparsity=ratio,
                                       ignored_layers=[m.conv_out])
    base_macs, base_params = tp.utils.count_ops_and_params(m, example)
    groups = []
    for g in pruner.step(interactive=True):
        module, fn = g[0][0].target.module, g[0][0].handler
        cur = pruner.DG.get_out_channels(module)
        full = pruner.DG.get_pruning_group(module, fn, list(range(cur)))
        ch_groups = pruner.get_channel_groups(full)
        sc = imp(full, ch_groups=ch_groups)
        groups.append({"root": names[module], "root_kind": KIND[fn], "ch_groups": int(ch_groups), "channels": int(cur),
                       "items": [(n, k, compress(i)) for n, k, i in describe_group(full, names)],
                       "imp": sc.clone(), "idxs": [int(i) for i in g[0][1]]})
        g.prune()
    for mod in m.modules():
        if isinstance(mod, (Upsample2D, Downsample2D)):
            mod.channels = mod.conv.in_channels
    macs, params = tp.utils.count_ops_and_params(m, example)
    res = {"cfg": cfg, "ratio": ratio, "groups": groups, "base": [base_macs, base_params], "pruned": [macs, params],
           "pruned_shapes": {k: list(v.shape) for k, v in m.state_dict().items()}}
    torch.save(res, os.path.join(OUT, "lsun_struct_magnitude.pt"))
    print("lsun_struct", len(groups), base_params, params, base_macs, macs)


def gen_exp_importance():
    """The ddpm_exp importance criteria (ddpm_exp/torch_pruning/importance.py:438-548 FullTaylor order 1/2, :553-670 AbsTaylor,
    :672-781 Fisher) evaluated by the UNMODIFIED vendored classes on every pruning group of the TINY UNet after two accumulated passes."""
    os.chdir("/tmp")
    cfg = dict(dp.TINY_TEST_CONFIG)
    m = build(cfg)
    sched = DDPMScheduler(num_train_timesteps=1000)
    clean, noise = inputs(2, 16)
    m.zero_grad()
    for tt in (7, 400):
        t = (tt * torch.ones(2)).long()
        torch.nn.functional.mse_loss(m(sched.add_noise(clean, noise, t), t).sample, noise).backward()
    example = {"sample": torch.randn(1, 3, 16, 16), "timestep": torch.ones((1,)).long()}
    pruner = tp.pruner.MagnitudePruner(m, example, importance=tp.importance.MagnitudeImportance(), iterative_steps=1, channel_groups={},
                                       ch_sparsity=0.3, ignored_layers=[m.conv_out])
    names = {mod: n for n, mod in m.named_modules()}
    crits = {"full1": tp.importance.FullTaylorImportance(order=1), "full2": tp.importance.FullTaylorImportance(order=2),
             "abs": tp.importance.AbsTaylorImportance(), "fisher": tp.importance.FisherImportance()}
    groups = []
    for g in pruner.DG.get_all_groups(ignored_layers=pruner.ignored_layers, root_module_types=pruner.root_module_types):
        items = describe_group_c(g, names)
        groups.append({"root": names[g[0][0].target.module], "items": items,
                       "imp": {k: c(g).clone() for k, c in crits.items()}})
    torch.save({"cfg": cfg, "groups": groups}, os.path.join(OUT, "exp_importance_tiny.pt"))
    print("exp_importance", len(groups), os.path.getsize(os.path.join(OUT, "exp_importance_tiny.pt")))


def gen_ldm_tiny():
    """The latent-diffusion UNetModel (BASELINE configs[4]) from the UNMODIFIED reference modules
    (ldm_exp/ldm/modules/diffusionmodules/openaimodel.py + ldm_exp/ldm/modules/attention.py; omegaconf is stubbed, openaimodel.py:476):
    a small member of the cin256-v2 family whose zero-initialised convolutions are re-drawn (a random-init network otherwise outputs 0
    and back-propagates nothing into most layers): state-dict keys, eps_hat, loss and all gradients after two accumulated Taylor passes
    (q_sample with the LDM sqrt-linear schedule, mse loss — what `get_loss_at_t` returns, ddpm.py:881-889,1022-1056); plus the parameter
    count of the full cin256-v2 network."""
    import types
    sys.path.insert(0, os.path.join(ref_shim.REF, "ldm_exp"))
    oc, lc = types.ModuleType("omegaconf"), types.ModuleType("omegaconf.listconfig")
    lc.ListConfig = type("ListConfig", (list,), {})
    oc.listconfig = lc
    sys.modules.setdefault("omegaconf", oc)
    sys.modules.setdefault("omegaconf.listconfig", lc)
    from ldm.modules.diffusionmodules.openaimodel import UNetModel as RefUNet
    from diff_pruning_b200 import ldm as L
    cfg = dict(L.LDM_TINY_CONFIG)
    torch.manual_seed(0)
    m = RefUNet(**cfg).eval()
    g = torch.Generator().manual_seed(5)
    redrawn = []
    for k, p in m.named_parameters():
        if float(p.detach().abs().sum()) == 0 and p.dim() > 1:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.05)
            redrawn.append(k)
    betas = torch.linspace(0.0015 ** 0.5, 0.0195 ** 0.5, 1000, dtype=torch.float64) ** 2
    ac = torch.cumprod(1.0 - betas, dim=0).to(torch.float32)
    clean, noise = inputs(2, 16)
    ctx = torch.randn(2, 1, cfg["context_dim"], generator=g)
    m.zero_grad()
    losses = []
    for tt in (7, 400):
        t = (tt * torch.ones(2)).long()
        xt = (ac[t] ** 0.5).reshape(-1, 1, 1, 1) * clean + ((1 - ac[t]) ** 0.5).reshape(-1, 1, 1, 1) * noise
        out = m(xt, t, context=ctx)
        loss = torch.nn.functional.mse_loss(out, noise)
        loss.backward()
        losses.append(loss.item())
    torch.manual_seed(0)
    n_full = sum(p.numel() for p in RefUNet(**L.CIN256_V2_CONFIG).parameters())
    import hashlib
    sha = hashlib.sha256(b"".join(v.detach().numpy().tobytes() for v in m.state_dict().values())).hexdigest()
    # weights are reproducible (seed 0 construction + the redraw loop above with Generator(5), context drawn right after): only their digest is stored
    torch.save({"cfg": cfg, "redrawn": redrawn, "sd_keys": list(m.state_dict().keys()), "sd_sha": sha, "context": ctx, "losses": losses,
                "out_last": out.detach(), "grads": {k: p.grad.clone() for k, p in m.named_parameters()}, "alphas_cumprod_fp": fp(ac),
                "cin256_v2_params": n_full}, os.path.join(OUT, "ldm_tiny.pt"))
    print("ldm_tiny", losses, n_full, len(redrawn), os.path.getsize(os.path.join(OUT, "ldm_tiny.pt")))


LDM_DDIM_RUNS = [(S, scale, eta) for S in (4, 20) for scale in (1.0, 3.0) for eta in (0.0, 0.5)]


def gen_ldm_ddim():
    """prune_ldm.py's sample-then-score loop on the tiny LDM (tests/golden/ldm_ddim_tiny.pt), from the UNMODIFIED reference: its DDIMSampler
    (ldm/models/diffusion/ddim.py, with register_buffer keeping the buffers on the CPU, ref_shim.cpu_ddim_sampler), its UNetModel (weights as
    gen_ldm_tiny makes them) and its ClassEmbedder (ldm/modules/encoders/modules.py:21-33, seed 1) behind a shim with LatentDiffusion's
    schedule buffers (ddpm.py:117-145, cin256-v2: linear 0.0015..0.0195, 1000 steps) and apply_model (crossattn context).
    One 3 x 8 x 8 latent per sample (2 images per guided forward) (small enough to keep the file small; 64 / 16 tokens in the two transformer levels).  Per run
    (S, scale, eta) with a fixed x_T and torch.manual_seed(20 + run) for the sigma noise: the DDIM timesteps and schedule arrays as
    make_schedule leaves them (dtype included), the samples and the intermediates at log_every_t = 5; for the 4-step runs and the 20-step
    scale-3 eta-0.5 run also every step's raw UNet output (the 2B batch when guided), x_prev and pred_x0.  Then one get_loss_at_t
    (p_losses, ddpm.py:1022-1056, restated: eps, l2, logvar 0, no elbo term) at t = 5 on the S = 20, scale 3, eta 0 samples with seeded
    noise: the loss, the UNet output, (sum, sum |g|, sum g^2) of every UNet gradient and its first 32 elements.  The embedding weights
    are reproducible (seed 1): only their digest is stored."""
    import functools
    import numpy as np
    ref_shim.install_ldm()
    from ldm.modules.diffusionmodules.openaimodel import UNetModel as RefUNet
    from ldm.modules.diffusionmodules.util import make_beta_schedule
    from ldm.modules.encoders.modules import ClassEmbedder as RefClassEmbedder
    from diff_pruning_b200 import ldm as L
    cfg = dict(L.LDM_TINY_CONFIG)
    torch.manual_seed(0)
    unet = RefUNet(**cfg).eval()
    g = torch.Generator().manual_seed(5)
    for k, p in unet.named_parameters():
        if float(p.detach().abs().sum()) == 0 and p.dim() > 1:
            p.data.copy_(torch.randn(p.shape, generator=g) * 0.05)
    torch.manual_seed(1)
    emb = RefClassEmbedder(cfg["context_dim"], n_classes=1001, key="class_label")

    class Shim:
        """LatentDiffusion's attributes that DDIMSampler reads (ddpm.py:117-145 register_schedule, :901-924 apply_model)."""
        num_timesteps, device = 1000, torch.device("cpu")

        def __init__(self):
            betas = make_beta_schedule("linear", 1000, linear_start=0.0015, linear_end=0.0195)
            ac = np.cumprod(1. - betas, axis=0)
            to_torch = functools.partial(torch.tensor, dtype=torch.float32)
            self.betas, self.alphas_cumprod = to_torch(betas), to_torch(ac)
            self.alphas_cumprod_prev = to_torch(np.append(1., ac[:-1]))
            self.sqrt_alphas_cumprod, self.sqrt_one_minus_alphas_cumprod = to_torch(np.sqrt(ac)), to_torch(np.sqrt(1. - ac))
            self.raw = []

        def apply_model(self, x, t, cond):
            out = unet(x, t, context=cond)
            self.raw.append(out.detach().clone())
            return out

    shim = Shim()
    Sampler = ref_shim.cpu_ddim_sampler()
    B = 1
    labels, ulabels = torch.tensor([998]), torch.tensor([1000])
    with torch.no_grad():
        c, uc = emb({"class_label": labels}), emb({"class_label": ulabels})
    HW = 8
    x_T = torch.randn(B, 3, HW, HW, generator=torch.Generator().manual_seed(7))

    def arr(v):
        return {"value": torch.as_tensor(np.asarray(v) if not torch.is_tensor(v) else v).clone(), "type": type(v).__name__,
                "dtype": str(v.dtype)}

    runs = {}
    for k, (S, scale, eta) in enumerate(LDM_DDIM_RUNS):
        steps = []

        class Rec(Sampler):
            def p_sample_ddim(self, x, c_, t, index, **kw):
                n0 = len(shim.raw)
                x_prev, pred_x0 = super().p_sample_ddim(x, c_, t, index, **kw)
                if S == 4 or (scale, eta) == (3.0, 0.5):
                    steps.append({"t": int(t[0]), "index": index, "raw": shim.raw[n0].clone(), "x_prev": x_prev.clone(),
                                  "pred_x0": pred_x0.clone()})
                return x_prev, pred_x0

        sampler = Rec(shim)
        torch.manual_seed(20 + k)
        samples, inter = sampler.sample(S=S, batch_size=B, shape=[3, HW, HW], conditioning=c, verbose=False, eta=eta, x_T=x_T.clone(),
                                        log_every_t=5, unconditional_guidance_scale=scale, unconditional_conditioning=uc)
        sched = {n: arr(getattr(sampler, n)) for n in ("ddim_timesteps", "ddim_alphas", "ddim_alphas_prev", "ddim_sigmas",
                                                       "ddim_sqrt_one_minus_alphas")}
        # the per-step fp32 scalars p_sample_ddim forms (ddim.py:190-193: torch.full of one entry of each array)
        full = {n: torch.tensor([float(torch.full((1,), getattr(sampler, a)[i]).item()) for i in range(S)], dtype=torch.float32)
                for n, a in (("a_t", "ddim_alphas"), ("a_prev", "ddim_alphas_prev"), ("sigma_t", "ddim_sigmas"),
                             ("sqrt_one_minus_at", "ddim_sqrt_one_minus_alphas"))}
        x_inter = torch.stack(inter["x_inter"])
        logged = [next(i for i, s in enumerate(steps) if torch.equal(s["x_prev"], v)) for v in x_inter[1:]] if steps else None
        packed = {f: torch.stack([st[f] for st in steps]) for f in ("raw", "x_prev", "pred_x0")} if steps else None
        if packed:                      # one stacked tensor per field: per-tensor records would outweigh the data
            packed.update({f: torch.tensor([st[f] for st in steps]) for f in ("t", "index")})
        runs[(S, scale, eta)] = {"seed": 20 + k, "sched": sched, "full": full, "steps": packed, "samples": samples.clone(),
                                 "x_inter": x_inter, "logged_steps": logged}
        shim.raw.clear()
        print("ldm_ddim", S, scale, eta, float(samples.abs().max()), logged)

    x0 = runs[(20, 3.0, 0.0)]["samples"]
    noise = torch.randn(x0.shape, generator=torch.Generator().manual_seed(11))
    t = torch.full((B,), 5, dtype=torch.long)
    unet.zero_grad()
    emb.zero_grad()
    cond = emb({"class_label": labels})
    ex = lambda a: a.gather(-1, t).reshape(B, 1, 1, 1)           # util.py extract_into_tensor
    x_noisy = ex(shim.sqrt_alphas_cumprod) * x0 + ex(shim.sqrt_one_minus_alphas_cumprod) * noise
    out = unet(x_noisy, t, context=cond)
    loss = ((out - noise) ** 2).mean([1, 2, 3])
    logvar_t = torch.zeros(1000)[t]
    loss = 1.0 * (loss / torch.exp(logvar_t) + logvar_t).mean()
    loss.backward()
    torch.save({"cfg": cfg, "runs_keys": LDM_DDIM_RUNS, "runs": runs, "x_T": x_T, "labels": labels, "ulabels": ulabels,
                "embedding_sha": hashlib.sha256(emb.embedding.weight.detach().numpy().tobytes()).hexdigest(),
                "emb_keys": list(emb.state_dict().keys()),
                "schedule": {"betas": shim.betas, "alphas_cumprod": shim.alphas_cumprod, "alphas_cumprod_prev": shim.alphas_cumprod_prev},
                "loss_t": 5, "loss_noise": noise, "loss": float(loss), "loss_out": out.detach(),
                "grad_names": [k for k, _ in unet.named_parameters()],
                "grad_samples": torch.stack([torch.nn.functional.pad(p.grad.flatten()[:32], (0, max(0, 32 - p.numel())))
                                             for p in unet.parameters()]),
                "grad_numel": torch.tensor([p.numel() for p in unet.parameters()]),
                "grad_fp": torch.tensor([fp(p.grad) for p in unet.parameters()], dtype=torch.float64),
                "emb_grad_fp": fp(emb.embedding.weight.grad)},
               os.path.join(OUT, "ldm_ddim_tiny.pt"))
    print("ldm_ddim loss", float(loss), os.path.getsize(os.path.join(OUT, "ldm_ddim_tiny.pt")))


def gen_ref_pickle():
    """A whole-module pickle exactly as the reference writes it (`torch.save(model)`, ddpm_prune.py:135) for a small member of the
    family after a `--pruner magnitude` prune at ratio 0.3 — default AttnProcessor2_0 objects, FrozenDict config and all — plus eps_hat
    of that network (legacy processor, the only one that runs on pruned widths).  Pins `torch.load(pruned_ckpt)` at ddpm_train.py:292
    / ddpm_sample.py:27 against this package's classes."""
    os.chdir("/tmp")
    cfg = dict(dp.TINY_TEST_CONFIG, block_out_channels=(16, 32))
    torch.manual_seed(0)
    m = UNet2DModel(**cfg).eval()
    example = {"sample": torch.randn(1, 3, 16, 16), "timestep": torch.ones((1,)).long()}
    pruner = tp.pruner.MagnitudePruner(m, example, importance=tp.importance.MagnitudeImportance(), iterative_steps=1,
                                       channel_groups={}, ch_sparsity=0.3, ignored_layers=[m.conv_out])
    for g in pruner.step(interactive=True):
        g.prune()
    for mod in m.modules():
        if isinstance(mod, (Upsample2D, Downsample2D)):
            mod.channels = mod.conv.in_channels
    m.zero_grad()
    del pruner
    torch.save(m, os.path.join(OUT, "ref_pruned_small.pth"))
    legacy_attn(m)
    sched = DDPMScheduler(num_train_timesteps=1000)
    clean, noise = inputs(2, 16)
    t = torch.tensor([3, 950]).long()
    with torch.no_grad():
        out = m(sched.add_noise(clean, noise, t), t).sample
    torch.save({"cfg": cfg, "t": t, "eps": out, "shapes": {k: list(v.shape) for k, v in m.state_dict().items()},
                "scales": {n: float(a.scale) for n, a in m.named_modules() if isinstance(a, Attention)}},
               os.path.join(OUT, "ref_pruned_small_out.pt"))
    print("ref_pickle", os.path.getsize(os.path.join(OUT, "ref_pruned_small.pth")), sum(p.numel() for p in m.parameters()))


def gen_fid():
    """FID fixtures from the UNMODIFIED inception.py / fid_score.py.  The weights are a seeded random state dict
    (oracle.inception_oracle.seeded_state_dict): inception.py's module-level load_state_dict_from_url is replaced, before any
    InceptionV3 is built, by a function returning it, so nothing is fetched.  Writes
      fid_weights.json  the weight file's keys and shapes (torchvision names), the wrapper's keys, the seeded state dict's digest
      fid_features.pt   uint8 input images (32x32, 64x64, 256x256) and their pool features for all four output blocks
      fid_frechet.pt    (mu1, sigma1, mu2, sigma2) -> calculate_frechet_distance, including a product that takes the singular branch"""
    import numpy as np
    import torchvision.transforms as TF
    from scipy import linalg
    from oracle import inception_oracle as orc
    import inception as ref_inception

    tv = ref_inception._inception_v3(num_classes=1008, aux_logits=False, weights=None)
    for name, block in (("Mixed_5b", ref_inception.FIDInceptionA(192, pool_features=32)),
                        ("Mixed_5c", ref_inception.FIDInceptionA(256, pool_features=64)),
                        ("Mixed_5d", ref_inception.FIDInceptionA(288, pool_features=64)),
                        ("Mixed_6b", ref_inception.FIDInceptionC(768, channels_7x7=128)),
                        ("Mixed_6c", ref_inception.FIDInceptionC(768, channels_7x7=160)),
                        ("Mixed_6d", ref_inception.FIDInceptionC(768, channels_7x7=160)),
                        ("Mixed_6e", ref_inception.FIDInceptionC(768, channels_7x7=192)),
                        ("Mixed_7b", ref_inception.FIDInceptionE_1(1280)), ("Mixed_7c", ref_inception.FIDInceptionE_2(2048))):
        setattr(tv, name, block)
    shapes = [(k, list(v.shape)) for k, v in tv.state_dict().items()]
    seeded = orc.seeded_state_dict(shapes, seed=0)

    def offline_loader(url, *a, **kw):
        assert url == ref_inception.FID_WEIGHTS_URL
        return {k: v.clone() for k, v in seeded.items()}
    ref_inception.load_state_dict_from_url = offline_loader
    net = ref_inception.InceptionV3([0, 1, 2, 3]).eval()
    json.dump({"weight_file": shapes, "wrapper": [(k, list(v.shape)) for k, v in net.state_dict().items()],
               "seed": 0, "digest": orc.state_dict_digest(seeded)}, open(os.path.join(OUT, "fid_weights.json"), "w"))

    g = torch.Generator().manual_seed(1)
    images = {hw: torch.randint(0, 256, (2, hw, hw, 3), dtype=torch.uint8, generator=g) for hw in (32, 64, 256)}
    feats = {}
    with torch.no_grad():
        for hw, u8 in images.items():
            x = torch.stack([TF.ToTensor()(im.numpy()) for im in u8])      # fid_score.py:129 on HWC uint8, as PIL decoding yields
            outs = net(x)
            feats[hw] = [orc.pooled(o) for o in outs]
            print("fid features", hw, [f"{float(f.abs().mean()):.3g}" for f in feats[hw]])
    torch.save({"images": images, "features": feats}, os.path.join(OUT, "fid_features.pt"))

    # fid_score.py calls sqrtm(..., disp=False), which scipy >= 1.16 no longer takes: give it that form back for the generator only
    sqrtm = linalg.sqrtm

    def sqrtm_disp(a, disp=True):
        r = sqrtm(a)
        return (r, 0.0) if not disp else r
    linalg.sqrtm = sqrtm_disp
    import fid_score as ref_fid
    rng = np.random.default_rng(2)
    cases = []
    for n, d in ((50, 8), (40, 16)):
        a, b = rng.standard_normal((n, d)), rng.standard_normal((n, d)) * 1.5 + 0.3
        case = dict(mu1=a.mean(0), sigma1=np.cov(a, rowvar=False), mu2=b.mean(0), sigma2=np.cov(b, rowvar=False))
        case["fid"] = float(ref_fid.calculate_frechet_distance(**case))
        cases.append(case)
    # sigma1 sigma2 = [[0, 1], [0, 0]] has no square root: the eps-offset retry runs, and its complex root fails the imaginary check
    case = dict(mu1=np.zeros(2), sigma1=np.array([[0.0, 1.0], [1.0, 0.0]]), mu2=np.ones(2), sigma2=np.diag([0.0, 1.0]))
    try:
        case["fid"] = float(ref_fid.calculate_frechet_distance(**case))
    except ValueError as e:
        case["error"] = str(e)
    cases.append(case)
    linalg.sqrtm = sqrtm
    torch.save(cases, os.path.join(OUT, "fid_frechet.pt"))
    print("fid frechet", [c.get("fid", c.get("error")) for c in cases])


def gen_ssim():
    """SSIM fixtures from the UNMODIFIED ldm_exp/ldm/modules/image_degradation/utils_image.py (fp64 NumPy + cv2: 11-tap Gaussian,
    sigma 1.5, valid region, C1 = (0.01 * 255)^2, C2 = (0.03 * 255)^2), loaded by file path so that ldm/__init__ is not imported.
    Writes ssim_ref.pt: a list of seeded uint8 HWC image pairs, each with the reference's per-channel ssim() and calculate_ssim()."""
    import importlib.util
    import numpy as np
    path = os.path.join(ref_shim.REF, "ldm_exp", "ldm", "modules", "image_degradation", "utils_image.py")
    spec = importlib.util.spec_from_file_location("ref_utils_image", path)
    ui = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ui)
    rng = np.random.default_rng(4)

    def u8(a):
        return np.clip(np.rint(a), 0, 255).astype(np.uint8)

    def smooth(h, w):
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing="ij")
        ph = rng.uniform(0, 2 * np.pi, 3)
        return np.stack([128 + 90 * np.sin(2 * np.pi * (1.3 * xx + 0.7 * yy) + ph[c]) * np.cos(3 * yy + c) for c in range(3)], -1)

    pairs = []
    noise = rng.integers(0, 256, (32, 32, 3))
    pairs.append(("noise", u8(noise), u8(rng.integers(0, 256, (32, 32, 3)))))
    s = smooth(32, 32)
    pairs.append(("smooth_vs_noisy", u8(s), u8(s + rng.normal(0, 4, s.shape))))
    flat = np.full((32, 32, 3), 100.0)
    pairs.append(("flat_vs_flat_plus_1", u8(flat), u8(flat + 1)))     # zero variance: the moments cancel exactly down to C2
    pairs.append(("inverted", u8(s), u8(255 - s)))
    pairs.append(("identical", u8(noise), u8(noise)))
    s = smooth(48, 40)
    pairs.append(("nonsquare_48x40", u8(s), u8(s + rng.normal(0, 8, s.shape))))
    s = smooth(256, 256)
    pairs.append(("smooth_256", u8(s), u8(s + rng.normal(0, 6, s.shape))))
    out = []
    for name, x, y in pairs:
        per_c = [float(ui.ssim(x[:, :, c], y[:, :, c])) for c in range(3)]
        out.append({"name": name, "x": torch.from_numpy(x), "y": torch.from_numpy(y), "ssim_c": torch.tensor(per_c, dtype=torch.float64),
                    "ssim": float(ui.calculate_ssim(x, y))})
        print("ssim", name, x.shape, per_c, out[-1]["ssim"])
    torch.save(out, os.path.join(OUT, "ssim_ref.pt"))
    print("ssim_ref.pt", os.path.getsize(os.path.join(OUT, "ssim_ref.pt")))


VQ_TINY_DDCONFIG = dict(double_z=False, z_channels=3, resolution=16, in_channels=3, out_ch=3, ch=64, ch_mult=(1, 2), num_res_blocks=1,
                        attn_resolutions=(), dropout=0.0)


def gen_vq_decoder():
    """The LDM's VQ first-stage Decoder from the UNMODIFIED reference module (ldm_exp/ldm/modules/diffusionmodules/model.py, imported
    through ref_shim.install_ldm): for a small config (2 levels, 64 channels, 8 x 8 latent) and the full cin256-v2 VQ-f4 ddconfig at a
    16 x 16 latent (64 x 64 output, 256 attention tokens), the state-dict keys, the seed and digest of the seed-s weights (torch.manual_seed(s);
    Decoder(**cfg)), two seeded latents and the reference outputs; plus the nearest-code choices of the cdist formula
    (diffusers/models/vae.py:338) and of taming's VectorQuantizer2 formula as recalled (z^2 + e^2 - 2 z e^T; taming is not in the reference
    tree) for a seeded latent against a seeded 8192 x 3 codebook."""
    ref_shim.install_ldm()
    from ldm.modules.diffusionmodules.model import Decoder as RefDecoder
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    from oracle import vq_oracle as vo
    out = {"configs": {}}
    for name, ddcfg, hw, seed in (("tiny", VQ_TINY_DDCONFIG, 8, 0), ("vq_f4", dict(VQ_F4_CONFIG["ddconfig"]), 16, 1)):
        torch.manual_seed(seed)
        dec = RefDecoder(**ddcfg).eval()
        sd = dec.state_dict()
        g = torch.Generator().manual_seed(100 + seed)
        z = torch.randn(2, ddcfg["z_channels"], hw, hw, generator=g)
        with torch.no_grad():
            y = dec(z)
        out["configs"][name] = {"ddconfig": ddcfg, "seed": seed, "sd_keys": list(sd.keys()), "digest": vo.state_dict_digest(sd),
                                "z": z, "out": y.detach()}
        print("vq_decoder", name, tuple(y.shape), float(y.abs().max()))
    g = torch.Generator().manual_seed(7)
    code = (torch.rand(8192, 3, generator=g) * 2 - 1) / 8192 * 64
    z = torch.randn(4096, 3, generator=g) * 0.004
    out["codes"] = {"codebook_seed": 7, "z": z, "cdist": vo.nearest_code_cdist(z, code), "taming": vo.nearest_code_taming(z, code)}
    torch.save(out, os.path.join(OUT, "vq_decoder_tiny.pt"))
    print("vq_decoder_tiny.pt", os.path.getsize(os.path.join(OUT, "vq_decoder_tiny.pt")))


def gen_vq_encoder():
    """The LDM's VQ first-stage encode side from the UNMODIFIED reference modules (ldm_exp/ldm/modules/diffusionmodules/model.py's
    Encoder, ldm/models/autoencoder.py's VQModelInterface through ref_shim.install_vq_model) for the small decoder-fixture config (16 x 16
    images) and the cin256-v2 VQ-f4 ddconfig (64 x 64 images, the size of a cin256-v2 latent sample: 16 x 16 output, 256 attention
    tokens): the state-dict keys and digests of the seed-s Encoder (torch.manual_seed(s); Encoder(**cfg)) and of the seed-s
    VQModelInterface (lossconfig torch.nn.Identity, as cin256-v2), two seeded inputs in [-1, 1] and the reference outputs of
    Encoder.forward and VQModelInterface.encode."""
    ref_shim.install_vq_model()
    from ldm.models.autoencoder import VQModelInterface as RefVQ
    from ldm.modules.diffusionmodules.model import Encoder as RefEncoder
    from diff_pruning_b200.autoencoder import VQ_F4_CONFIG
    from oracle import vq_oracle as vo
    out = {"configs": {}}
    for name, ddcfg, hw, n_embed, seed in (("tiny", VQ_TINY_DDCONFIG, 16, 64, 0), ("vq_f4", dict(VQ_F4_CONFIG["ddconfig"]), 64, 8192, 1)):
        torch.manual_seed(seed)
        enc = RefEncoder(**ddcfg).eval()
        torch.manual_seed(seed)
        vq = RefVQ(embed_dim=ddcfg["z_channels"], n_embed=n_embed, ddconfig=ddcfg, lossconfig={"target": "torch.nn.Identity"}).eval()
        g = torch.Generator().manual_seed(200 + seed)
        x = torch.rand(2, ddcfg["in_channels"], hw, hw, generator=g) * 2 - 1
        with torch.no_grad():
            y, z = enc(x), vq.encode(x)
        out["configs"][name] = {"ddconfig": ddcfg, "seed": seed, "n_embed": n_embed, "hw": hw,
                                "sd_keys": list(enc.state_dict().keys()), "digest": vo.state_dict_digest(enc.state_dict()),
                                "vq_sd_keys": list(vq.state_dict().keys()), "vq_digest": vo.state_dict_digest(vq.state_dict()),
                                "x": x, "out": y.detach(), "encoded": z.detach()}
        print("vq_encoder", name, tuple(z.shape), float(y.abs().max()), float(z.abs().max()))
    torch.save(out, os.path.join(OUT, "vq_encoder_tiny.pt"))
    print("vq_encoder_tiny.pt", os.path.getsize(os.path.join(OUT, "vq_encoder_tiny.pt")))


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-cfg1", action="store_true")
    ap.add_argument("--only", default=None)
    a = ap.parse_args()
    torch.set_num_threads(os.cpu_count())
    jobs = {"vq_encoder": gen_vq_encoder, "vq_decoder": gen_vq_decoder, "ssim": gen_ssim, "fid": gen_fid,"ldm_tiny": gen_ldm_tiny, "ldm_ddim": gen_ldm_ddim, "exp_importance": gen_exp_importance, "ref_pickle": gen_ref_pickle, "lsun_struct": gen_lsun_struct, "lr": gen_lr, "ckpt": gen_ckpt, "ddim": gen_ddim, "tiny": gen_tiny, "blocks": gen_blocks, "finetune": gen_finetune, "cifar_fwd": gen_cifar_fwd,
            "cfg1_s3": gen_cfg1_s3, "cfg3_s3": gen_cfg3_s3, "cfg1": gen_cfg1}
    for name, fn in jobs.items():
        if a.only and name != a.only:
            continue
        if name.startswith("cfg") and a.skip_cfg1:
            continue
        fn()
