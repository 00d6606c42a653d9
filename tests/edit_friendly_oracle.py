"""CPU restatement of the edit-friendly inversion on the lock-step cycle (test infrastructure only).

The reference has no edit-friendly inversion, so this is pinned by its definition (include/cdx.h, cdx_cycle_lockstep_sampler) and,
in tests/test_edit_friendly_cpu.py, by float64 algebra: a first-order SDE-DPM-Solver++ step is the DDIM eta = 1 step, and with
identical chains the loop hands the target the source's draws back.

  * latent_init / latent_step: latent_chains_init / latent_chains_step (kernels_elem.cu) under solver 1 and 2, in
    tests/step_oracle.py's conventions (flat buffers, chain tables, one fp32 torch op per kernel op).  The target chains' eps-hat is
    looked up as step_oracle._eps_hat at call time, so the SEGA / LEDITS++ test helpers that patch it drive this step too.
  * ef_cycle: the whole loop of UNet.cycle_lockstep under a schedule.EditFriendlySchedule, on any U-Net callable, in fp32 or (dtype
    float64, the tables' fp32 values widened) in float64.

Per step i with the source's draws x_k = qa[k]*x0 + q1[k]*noise[k] (x_R = x0), D a chain's x0-prediction:
    solver 1 ('ddpm'):        z = compute_eps(x_i, x_{i+1}, e, D);  y <- target_step(D_y, e_y, z)       (eta = 1 DDIM table)
    solver 2 ('dpmsolver++'): mu = a*x + b*D (+ c*(D - D_prev) at order 2);  z = (x_{i+1} - mu_src) / n;  y <- mu_y + n*z
then the mask blend with x_{i+1}.
"""
import torch

from tests import step_oracle as so
from tests.sega_oracle import _guided


def draw(x0, noise, qa, q1):
    """the source's independent draw: q_sample's op order, as x_T"""
    return so.x_T(x0, noise, qa, q1)


def dpm_mean(x, D, hist, dc, f=so.f):
    """a*x + b*D (+ c*(D - D_prev) at order 2); hist holds D_prev and takes D"""
    mu = f(dc.a) * x + f(dc.b) * D
    if dc.order == 2:
        mu = mu + f(dc.c) * (D - hist)
    hist.copy_(D)
    return mu


def latent_init(chains, chw, n_src, K, src, x0=None, noise0=None, sa=0.0, s1=0.0, xt=None, xn=None, next=0, noise_next=None,
                z_out=None, z_stride=0, eps_in=None, eps_stride=0, yt=None, xin=None, qa=0.0, q1=0.0, **_):
    """latent_chains_init under solver 1 and 2: next == 3 draws xn independently, next == 2 takes x0"""
    assert next in (0, 2, 3)
    for j in range(n_src):
        g = slice(j * chw, (j + 1) * chw)
        if src:
            x = so.x_T(x0[g], noise0[g], sa, s1)
            if z_out is not None:
                so._seg(z_out, j * z_stride, chw).copy_(x)
            xt[g] = x
            if next:
                xn[g] = draw(x0[g], noise_next[g], qa, q1) if next == 3 else x0[g]
            so._put(xin, chains[j], chw, x)
        else:
            x = so._seg(eps_in, j * eps_stride, chw)
        for k in range(K):
            t = j * K + k
            so._seg(yt, t * chw, chw).copy_(x)
            so._put(xin, chains[n_src + t], chw, x)


def latent_step(chains, chw, n_src, K, src, eout=None, c=None, x0=None, xt=None, xn=None, next=0, noise_next=None, xn2=None,
                z_out=None, z_stride=0, eps_in=None, eps_stride=0, yt=None, y_out=None, xin=None, pred=0, vsa=0.0, vs1=0.0, mask=None, hw=0,
                solver=1, dc=None, d_src=None, d_tgt=None, qa=0.0, q1=0.0, **_):
    """latent_chains_step under solver 1 (the DDIM step) or 2 (the SDE-DPM-Solver++ step under dc, histories d_src / d_tgt)"""
    assert solver in (1, 2) and next in (0, 2, 3)
    for j in range(n_src):
        g = slice(j * chw, (j + 1) * chw)
        if src:
            e_t, pred_x0 = so.eps_x0(so._eps_hat(eout, chains[j], chw), xt[g], c, pred, vsa, vs1)
            if solver == 2:
                eps = (xn[g] - dpm_mean(xt[g], pred_x0, d_src[g], dc)) / so.f(dc.n)
            else:
                eps = so.compute_eps(xt[g], xn[g], e_t, pred_x0, c)
            if z_out is not None:
                so._seg(z_out, j * z_stride, chw).copy_(eps)
            if next:
                xn2[g] = draw(x0[g], noise_next[g], qa, q1) if next == 3 else x0[g]
            so._put(xin, chains[j], chw, xn[g])
        else:
            eps = so._seg(eps_in, j * eps_stride, chw)
        m = so._seg(mask, j * hw, hw)[torch.arange(chw) % hw] if mask is not None else None
        for k in range(K):
            t = j * K + k
            y = so._seg(yt, t * chw, chw)
            e_t, pred_x0 = so.eps_x0(so._eps_hat(eout, chains[n_src + t], chw), y, c, pred, vsa, vs1)
            if solver == 2:
                yn = dpm_mean(y, pred_x0, so._seg(d_tgt, t * chw, chw), dc) + so.f(dc.n) * eps
            else:
                yn = so.target_step(pred_x0, e_t, eps, c)
            if m is not None:
                yn = so.blend(yn, xn[g], m)
            so._seg(y_out, t * chw, chw).copy_(yn)
            so._put(xin, chains[n_src + t], chw, yn)


def ef_cycle(unet_fn, x0, c_src, c_tgt, uc, sched, src_scale, tgt_scale, noise, mask=None, prediction='eps', v_tabs=None,
             dtype=torch.float32):
    """UNet.cycle_lockstep(x0, c_src, c_tgt, uc, src_scale, tgt_scale, sched, noise, return_z=True, mask=mask) under an
    EditFriendlySchedule: one source chain driving one target chain.  noise [R+1, B, C, h, w] as the pipeline draws it (noise[R]
    unused); prediction 'v' reads (sqrt(abar_t), sqrt(1 - abar_t)) from v_tabs at the step's timestep.  dtype float64 runs every op
    in float64 on the fp32 tables.  -> (target latent, z [B, R+1, C, h, w])."""
    f = lambda v: torch.full((1,), float(v), dtype=dtype)
    cast = lambda t: t.to(dtype) if t is not None else None
    x0, c_src, c_tgt, uc, noise, mask = (cast(t) for t in (x0, c_src, c_tgt, uc, noise, mask))
    R = sched.refine_steps
    xs = [f(sched.qa[k]) * x0 + f(sched.q1[k]) * noise[k] for k in range(R)] + [x0]     # draw()'s op order
    b = x0.shape[0]
    y, zs = xs[0], [xs[0]]
    hist_s, hist_t = torch.zeros_like(x0), torch.zeros_like(x0)
    for i in range(R):
        c, ts = sched.coef[i], torch.full((b,), int(sched.t_loop[i]), dtype=torch.long)
        vsa = vs1 = 0.0
        if prediction == 'v':
            vsa, vs1 = float(v_tabs[0][int(sched.t_loop[i])]), float(v_tabs[1][int(sched.t_loop[i])])

        def x0_pred(o, x):
            if prediction == 'eps':
                return o, (x - f(c.sqrt_1m_at_tab) * o) / f(c.sqrt_at)
            return f(vsa) * o + f(vs1) * x, f(vsa) * x - f(vs1) * o
        e_s, D_s = x0_pred(_guided(unet_fn, xs[i], ts, c_src, uc, src_scale)[0], xs[i])
        e_y, D_y = x0_pred(_guided(unet_fn, y, ts, c_tgt, uc, tgt_scale)[0], y)
        if sched.kind == 2:
            dc = sched.dpm[i]
            z = (xs[i + 1] - dpm_mean(xs[i], D_s, hist_s, dc, f)) / f(dc.n)
            y_new = dpm_mean(y, D_y, hist_t, dc, f) + f(dc.n) * z
        else:
            z = (xs[i + 1] - f(c.sqrt_aprev) * D_s - f(c.dir_coef) * e_s) / f(c.sigma) / 1.0
            y_new = f(c.sqrt_aprev) * D_y + f(c.dir_coef) * e_y + f(c.sigma) * z * 1.0
        zs.append(z)
        y = y_new if mask is None else so.blend(y_new, xs[i + 1], mask)
    return y, torch.stack(zs, dim=1)
