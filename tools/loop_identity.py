"""Bit-for-bit record of every latent loop entry point, for comparing two builds of libcdx on the same GPU.

    python tools/loop_identity.py --save FILE     # on the tree that is the reference
    python tools/loop_identity.py --check FILE    # on the tree under test: torch.equal on every tensor, exit 1 on a difference

Seeded inputs at a narrow U-Net topology: latent_encode, latent_decode (with and without extra noise), latent_refine,
cycle_lockstep, latent_encode_ens / latent_decode_ens at scales {0, 1, 3}, cycle_fan (mixed scales, K = 3) and latent_cycle_pair
(n_rec < refine_steps, on one and on two engines), each for eps- and v-prediction where the entry takes it; cycle_lockstep under
Prompt-to-Prompt control (replace with a non-identity token map and self control, refine with a nonzero own weight); one U-Net
call with 160-channel heads.  In mma modes 1 and 5 (fp16 planes) and 3 (TF32 planes), and beside every entry the number of
launches the engines enqueued for it.
"""
import argparse
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from cycle_diffusion_b200 import specs                    # noqa: E402
from cycle_diffusion_b200.attn_control import AttentionControl   # noqa: E402
from cycle_diffusion_b200.engine import Engine, UNet      # noqa: E402
from cycle_diffusion_b200.schedule import DDIMSchedule    # noqa: E402

COND = dict(in_channels=4, out_channels=4, model_channels=32, attention_resolutions=(4, 2, 1), num_res_blocks=2,
            channel_mult=(1, 2, 4, 4), num_heads=2, context_dim=48)
D160 = dict(in_channels=4, out_channels=4, model_channels=160, attention_resolutions=(1, 2), num_res_blocks=1, channel_mult=(1, 2),
            num_head_channels=160, context_dim=48)
UNCOND = dict(in_channels=3, out_channels=3, model_channels=32, attention_resolutions=(2, 4), num_res_blocks=1,
              channel_mult=(1, 2, 4), num_heads=2)


class Record(dict):
    """The recorded tensors and, under '<key>/launches', the launches the engines enqueued since the previous entry."""

    def __init__(self, *engines):
        super().__init__()
        self.engines, self.last = engines, 0

    def __setitem__(self, key, value):
        n = sum(e.launches for e in self.engines)
        super().__setitem__(key, value)
        super().__setitem__(f'{key}/launches', torch.tensor(n - self.last))
        self.last = n


def _unet(eng, cfg, seed):
    return UNet(eng, cfg, 'openai').load_state_dict(specs.synth_state_dict(specs.openai_unet_params(cfg), seed))


def _noise(g, n, shape, sched):
    """[n+1, *shape] in the encoder's draw order; the slot of the step that reaches index 0 draws nothing (ddim.py:583-584)."""
    noise = torch.randn(n + 1, *shape, generator=g)
    if n == sched.refine_steps:
        noise[n] = 0
    return noise


def conditional(eng, out, tag):
    unet = _unet(eng, COND, 11)
    g = torch.Generator().manual_seed(3)
    B = 3
    x0 = torch.randn(B, 4, 16, 16, generator=g) * 0.8
    c_src, c_tgt, uc = (torch.randn(B, 77, 48, generator=g) for _ in range(3))
    sched = DDIMSchedule(6, 0.1, 2)
    n = sched.refine_steps
    full, part = _noise(g, n, x0.shape, sched), _noise(g, n - 1, x0.shape, sched)
    extra = torch.randn(1, *x0.shape, generator=g)
    refine = torch.randn(3, *x0.shape, generator=g)
    mixed = [3.0, 0.0, 1.0]
    for pred in ('eps', 'v'):
        unet.set_prediction(pred)
        p = f'{tag}/{pred}/'
        for scale in (0.0, 1.0, 3.0):
            z = unet.latent_encode(x0, c_src, uc, scale, sched, n, full)
            out[f'{p}encode/{scale}'] = z
            out[f'{p}decode/{scale}'] = unet.latent_decode(z, c_tgt, uc, scale, sched)
            lat, zl = unet.cycle_lockstep(x0, c_src, c_tgt, uc, scale, 3.0 - scale, sched, full, return_z=True)
            out[f'{p}lockstep/{scale}/x'], out[f'{p}lockstep/{scale}/z'] = lat, zl
        out[f'{p}encode/no_uc'] = unet.latent_encode(x0, c_src, None, 3.0, sched, n, full)
        zp = unet.latent_encode(x0, c_src, uc, 3.0, sched, n - 1, part)
        out[f'{p}encode/partial'] = zp
        out[f'{p}decode/extra'] = unet.latent_decode(zp, c_tgt, uc, 3.0, sched, extra_noise=extra)
        out[f'{p}refine'] = unet.latent_refine(x0, c_tgt, uc, 3.0, 6, 2, refine)
        ze = unet.latent_encode_ens(x0, c_src, uc, mixed, sched, n, full)
        out[f'{p}encode_ens'] = ze
        out[f'{p}decode_ens'] = unet.latent_decode_ens(ze, c_tgt, uc, mixed[::-1], sched)
        out[f'{p}decode_ens/extra'] = unet.latent_decode_ens(zp, c_tgt, uc, mixed, sched, extra_noise=extra)
        lat, zf = unet.cycle_fan(x0, c_src, c_tgt, uc, mixed, [[1.0, 0.0, 3.0], [3.0, 2.0, 1.0], [0.0, 0.0, 5.0]], sched, full, return_z=True)
        out[f'{p}fan/x'], out[f'{p}fan/z'] = lat, zf
        L = c_src.shape[1]
        A = torch.eye(L).repeat(B, 1, 1)               # sample 1 swaps tokens 2 and 3, sample 2 spreads token 5 over 5 and 6
        A[1, 2, 2] = A[1, 3, 3] = 0.0
        A[1, 2, 3] = A[1, 3, 2] = 1.0
        A[2, 5, 5] = A[2, 5, 6] = 0.5
        A[2, 6, 6] = 0.0
        own = torch.zeros(B, L)
        own[:, 4] = 0.7                                # refine: token 4 has no source and keeps part of its own map
        A_ref = A.clone()
        A_ref[:, 4, 4] = 0.0
        for name, ctl in (('replace', AttentionControl(0.75, 0.5, self_max_tokens=64, token_map=A)),
                          ('refine', AttentionControl(0.75, 0.5, self_max_tokens=64, token_map=A_ref, own_weight=own))):
            lat, zl = unet.cycle_lockstep(x0, c_src, c_tgt, uc, 1.0, 3.0, sched, full, return_z=True, attn_control=ctl)
            out[f'{p}lockstep/{name}/x'], out[f'{p}lockstep/{name}/z'] = lat, zl


def heads160(eng, out, tag):
    unet = _unet(eng, D160, 13)
    g = torch.Generator().manual_seed(9)
    x = torch.randn(2, 4, 16, 16, generator=g)
    ctx = torch.randn(2, 77, 48, generator=g)
    out[f'{tag}/unet_d160'] = unet(x, torch.tensor([981., 21.]), ctx)


def pair(eng, eng2, out, tag):
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 16, 16, generator=g) * 0.8
    sched = DDIMSchedule(10, 0.1, 0)
    n_rec = 5
    noise = _noise(g, n_rec, x0.shape, sched)
    extra = torch.randn(sched.refine_steps - n_rec, *x0.shape, generator=g)
    for name, e_tgt in (('one', eng), ('two', eng2)):
        src, tgt = _unet(eng, UNCOND, 41), _unet(e_tgt, UNCOND, 43)
        out[f'{tag}/pair/{name}'] = src.latent_cycle_pair(tgt, x0, sched, n_rec, noise, extra_noise=extra)
        out[f'{tag}/pair/{name}/full'] = src.latent_cycle_pair(tgt, x0, sched, sched.refine_steps, _noise(g, sched.refine_steps, x0.shape, sched))


def main():
    ap = argparse.ArgumentParser()
    how = ap.add_mutually_exclusive_group(required=True)
    how.add_argument('--save')
    how.add_argument('--check')
    args = ap.parse_args()
    eng, eng2 = Engine(0), Engine(0)
    out = Record(eng, eng2)
    for mode in (1, 5, 3):
        eng.set_mma_mode(mode)
        eng2.set_mma_mode(mode)
        conditional(eng, out, f'mma{mode}')
        pair(eng, eng2, out, f'mma{mode}')
        if mode != 3:                                  # (TF32 planes at d = 160 keep the unfused route)
            heads160(eng, out, f'mma{mode}')
    torch.cuda.synchronize()
    out = {k: v.cpu() for k, v in out.items()}
    bad = [k for k, v in out.items() if not torch.isfinite(v).all()]
    assert not bad, f'non-finite outputs: {bad}'
    if args.save:
        torch.save(out, args.save)
        print(f'saved {len(out)} tensors to {args.save}')
        return 0
    ref = torch.load(args.check)
    diff = [k for k in sorted(set(ref) | set(out)) if k not in ref or k not in out or not torch.equal(ref[k], out[k])]
    for k in diff:
        d = float((ref[k].double() - out[k].double()).abs().max()) if k in ref and k in out and ref[k].shape == out[k].shape else float('nan')
        print(f'DIFFERENT {k}: max |d| {d:.3e}')
    print(f'{len(out) - len(diff)} of {len(out)} tensors bit-identical to {args.check}')
    return 1 if diff else 0


if __name__ == '__main__':
    sys.exit(main())
