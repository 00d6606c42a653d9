"""Host-side diffusion schedules, bit-replicating the reference's fp32 coefficient arithmetic.

The reference rebuilds these tables with (mixed numpy/torch) fp32 tensor ops on every call
(ddim.py:25-55, util.py:46-75; ddpm_ddim_wrapper.py:194-199, 264-303); the per-step kernels in libcdx take
the resulting fp32 scalars as arguments, so the tables must be produced with exactly the same sequence of
IEEE fp32 operations.  We therefore evaluate the very same expressions with torch CPU tensors of shape [1]
(PyTorch here is host-side plumbing; nothing in this file touches the GPU).
"""
import numpy as np
import torch

from ._cabi import DdimCoef, DpmCoef, PixelCoef, SamplerC


# ------------------------------------------------------------------------------------------ latent models
def ldm_alphas_cumprod(n_timestep=1000, linear_start=0.00085, linear_end=0.012):
    """make_beta_schedule('linear') (util.py:21-26) -> fp64 cumprod -> fp32 buffer (ddpm.py:117-138)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()
    return torch.tensor(np.cumprod(1.0 - betas, axis=0), dtype=torch.float32)


def ldm_alphas_cumprod_f64(n_timestep=1000, linear_start=0.00085, linear_end=0.012):
    """The same schedule before the fp32 cast: register_schedule's float64 alphas_cumprod (numpy)."""
    betas = (torch.linspace(linear_start ** 0.5, linear_end ** 0.5, n_timestep, dtype=torch.float64) ** 2).numpy()
    return np.cumprod(1.0 - betas, axis=0)


def v_tables(alphas_cumprod_f64=None):
    """The v-prediction tables of an SD 2 model, indexed by the U-Net timestep t: fp32(sqrt(abar_t)) and fp32(sqrt(1 - abar_t))
    of the float64 abar (register_schedule's sqrt_alphas_cumprod / sqrt_one_minus_alphas_cumprod buffers)."""
    ac = ldm_alphas_cumprod_f64() if alphas_cumprod_f64 is None else np.asarray(alphas_cumprod_f64, dtype=np.float64)
    return np.sqrt(ac).astype(np.float32), np.sqrt(1.0 - ac).astype(np.float32)


class DDIMSchedule:
    """DDIMSampler.make_schedule for (S, eta) plus the loop geometry of _ddpm_ddim_encoding / ddim_sampling_with_eps."""

    def __init__(self, S, eta, skip_steps=0, alphas_cumprod=None, num_ddpm_timesteps=1000):
        ac = ldm_alphas_cumprod(num_ddpm_timesteps) if alphas_cumprod is None else alphas_cumprod.to(torch.float32).cpu()
        assert ac.shape[0] == num_ddpm_timesteps, 'alphas have to be defined for each timestep'   # ddim.py:29
        c = num_ddpm_timesteps // S
        self.timesteps = np.asarray(list(range(0, num_ddpm_timesteps, c)))[:S] + 1            # util.py:46-61
        alphas = ac[self.timesteps]                                                          # fp32 torch
        alphas_prev = np.asarray([ac[0]] + ac[self.timesteps[:-1]].tolist())                 # fp64 numpy, util.py:67
        with np.errstate(all='ignore'):
            sigmas = eta * np.sqrt((1 - alphas_prev) / (1 - alphas) * (1 - alphas / alphas_prev))   # fp64 torch, util.py:70
            sqrt_1m = np.sqrt(1.0 - alphas)                                                      # fp32 torch, ddim.py:50
        self.total_steps = int(self.timesteps.shape[0])
        self.refine_steps = self.total_steps - skip_steps
        assert self.refine_steps >= 1
        self.eta = eta
        # loop order: iteration i uses index = refine_steps - 1 - i and timestep flip(timesteps)[-refine_steps:][i]
        time_range = np.flip(self.timesteps)[-self.refine_steps:]
        self.t_loop = [float(int(t)) for t in time_range]
        self.coef = []
        for i in range(self.refine_steps):
            index = self.refine_steps - 1 - i
            a_t = torch.full((1,), alphas[index])                      # ddim.py:570-573 (torch.full -> fp32)
            a_prev = torch.full((1,), alphas_prev[index])
            sigma_t = torch.full((1,), sigmas[index])
            s1m = torch.full((1,), sqrt_1m[index])
            self.coef.append(DdimCoef(
                sqrt_at=a_t.sqrt().item(),
                sqrt_1m_at=(1 - a_t).sqrt().item(),
                sqrt_1m_at_tab=s1m.item(),
                sqrt_aprev=a_prev.sqrt().item(),
                dir_coef=(1. - a_prev - sigma_t ** 2).sqrt().item(),
                sigma=sigma_t.item()))
        at = alphas[self.refine_steps - 1]                             # ddim.py:477-479
        self.sqrt_a_T = at.sqrt().item()
        self.sqrt_1ma_T = (1 - at).sqrt().item()

    def coef_array(self):
        return (DdimCoef * len(self.coef))(*self.coef)

    def t_array(self):
        import ctypes
        return (ctypes.c_float * len(self.t_loop))(*self.t_loop)


class EditFriendlySchedule(DDIMSchedule):
    """The edit-friendly inversion of LEDITS++ (Brack et al., 2024) on the DDIM schedule's timesteps and loop geometry, so strength
    and every step-counted control mean what they mean under DDIMSchedule.  solver 'ddpm': the independent draws stepped by the
    eta = 1 DDIM table (`coef`, inherited); 'dpmsolver++': the same draws stepped by the SDE-DPM-Solver++ table `dpm`, whose
    x0-prediction reads sqrt_at / sqrt_1m_at_tab from `coef`.
      qa[k], q1[k]  fp32 sqrt(abar) and sqrt(1 - abar) of loop step k's level, the source's draw x_k = qa[k]*x0 + q1[k]*noise
                    (the same torch fp32 expression as sqrt_a_T / sqrt_1ma_T, which are qa[0] / q1[0])
      dpm[i]        DpmCoef of step i from level s = abar(t_i) to level t = the DDIM table's a_prev of the step (abar[0] on the
                    last), formed in float64 from the fp32 abar and rounded once each (cdx.h, cdx_dpm_coef).  Order 1 on the first
                    step and, when the loop has fewer than 15 steps, on the last (diffusers' lower_order_final); else order 2."""
    SOLVERS = {'ddpm': 1, 'dpmsolver++': 2}      # cdx_sampler kinds CDX_SAMPLER_DDIM_DRAWS, CDX_SAMPLER_DPMSOLVER_DRAWS

    def __init__(self, S, skip_steps=0, alphas_cumprod=None, num_ddpm_timesteps=1000, solver='dpmsolver++'):
        if solver not in self.SOLVERS:
            raise ValueError(f"solver must be one of {sorted(self.SOLVERS)}, got {solver!r}")
        super().__init__(S, 1.0, skip_steps, alphas_cumprod, num_ddpm_timesteps)
        self.solver, self.kind = solver, self.SOLVERS[solver]
        ac = ldm_alphas_cumprod(num_ddpm_timesteps) if alphas_cumprod is None else alphas_cumprod.to(torch.float32).cpu()
        alphas = ac[self.timesteps]
        R = self.refine_steps
        self.qa, self.q1 = [], []
        for k in range(R):
            at = alphas[R - 1 - k]
            self.qa.append(at.sqrt().item())
            self.q1.append((1 - at).sqrt().item())
        self.dpm = [DpmCoef(**c) for c in self.dpm_table(ac, self.timesteps, R)]

    @staticmethod
    def dpm_table(ac, timesteps, R):
        """The SDE-DPM-Solver++ coefficients of the R loop steps as dicts (a, b, c, n, order), in float64 from the fp32 abar ac."""
        lev = [float(ac[timesteps[R - 1 - i]]) for i in range(R)] + [float(ac[0])]     # lev[i]: step i's level; lev[R]: abar[0]
        alpha = lambda v: np.sqrt(v)
        sigma = lambda v: np.sqrt(1.0 - v)
        lam = lambda v: np.log(alpha(v)) - np.log(sigma(v))
        out = []
        for i in range(R):
            s, t = lev[i], lev[i + 1]
            h = lam(t) - lam(s)
            em = -np.expm1(-2.0 * h)
            a = (sigma(t) / sigma(s)) * np.exp(-h)
            b = alpha(t) * em
            n = sigma(t) * np.sqrt(em)
            order = 1 if i == 0 or (i == R - 1 and R < 15) else 2
            c = 0.5 * b / ((lam(s) - lam(lev[i - 1])) / h) if order == 2 else 0.0
            out.append(dict(a=float(np.float32(a)), b=float(np.float32(b)), c=float(np.float32(c)), n=float(np.float32(n)), order=order))
        return out

    def sampler_struct(self):
        """-> (cdx_sampler, the host arrays it points to, which must outlive the call)"""
        import ctypes
        qa = (ctypes.c_float * len(self.qa))(*self.qa)
        q1 = (ctypes.c_float * len(self.q1))(*self.q1)
        dpm = (DpmCoef * len(self.dpm))(*self.dpm)
        sp = SamplerC(kind=self.kind, dpm=ctypes.cast(dpm, ctypes.POINTER(DpmCoef)), qa=ctypes.cast(qa, ctypes.POINTER(ctypes.c_float)),
                      q1=ctypes.cast(q1, ctypes.POINTER(ctypes.c_float)))
        return sp, (qa, q1, dpm)


def same_schedule(a, b):
    """Do two schedules drive identical loops: same kind and length, bit-identical coefficient tables, timesteps and x_T scalars?
    (Two models may then run their chains in lock-step.)"""
    return (type(a) is type(b) and getattr(a, 'es_steps', None) == getattr(b, 'es_steps', None) and a.t_loop == b.t_loop
            and (a.sqrt_a_T, a.sqrt_1ma_T) == (b.sqrt_a_T, b.sqrt_1ma_T) and len(a.coef) == len(b.coef)
            and all(bytes(x) == bytes(y) for x, y in zip(a.coef, b.coef)))


# ------------------------------------------------------------------------------------------ pixel models
class PixelSchedule:
    """Per-step scalars of DDPMDDIMWrapper.encode / generate (ddpm_ddim_wrapper.py:392-523)."""

    def __init__(self, sample_type, custom_steps, es_steps, eta=None, t_0=None, beta_start=1e-4, beta_end=2e-2, T=1000, var_type='fixedsmall'):
        if sample_type == 'ddim':
            assert eta > 0                                              # DW:333-334
        elif sample_type == 'ddpm':
            assert eta is None                                          # DW:335-336
        else:
            raise ValueError()
        self.sample_type, self.eta = sample_type, eta
        t_0 = 999 if t_0 is None else t_0
        betas64 = np.linspace(beta_start, beta_end, T, dtype=np.float64)            # diffusion_utils.py:5-9
        self.b = torch.from_numpy(betas64).float()                                   # DW:350-352
        ac = np.cumprod(1.0 - betas64, axis=0)
        ac_prev = np.append(1.0, ac[:-1])
        post_var = betas64 * (1.0 - ac_prev) / (1.0 - ac)
        if var_type == 'fixedlarge':                                                  # DW:362-363 (Ho-et-al checkpoints may use it)
            self.logvar = np.log(np.append(post_var[1], betas64[1:]))
        else:
            assert var_type == 'fixedsmall'
            self.logvar = np.log(np.maximum(post_var, 1e-20))                         # DW:356-373 (fp64)
        if (t_0 + 1) % custom_steps == 0:                                             # DW:393-400
            seq_inv = range(0, t_0 + 1, (t_0 + 1) // custom_steps)
            assert len(seq_inv) == custom_steps
        else:
            seq_inv = np.linspace(0, 1, custom_steps) * t_0
        seq_inv = [int(s) for s in list(seq_inv)][:es_steps]
        seq_inv_next = ([-1] + list(seq_inv[:-1]))[:es_steps]
        self.pairs = list(zip(reversed(seq_inv), reversed(seq_inv_next)))             # loop order (noisiest first)
        self.es_steps = es_steps
        self.cumprod = (1.0 - self.b).cumprod(dim=0)                                  # fp32, DW:194 (re-done per step there)
        at = self._extract(self.cumprod, es_steps - 1)                                # DW:483-484: es_steps-1 used as a timestep
        self.sqrt_a_T = at.sqrt().item()
        self.sqrt_1ma_T = (1 - at).sqrt().item()
        self.coef = [self.step_coef(i, j, eta) for i, j in self.pairs]
        self.t_loop = [float(i) for i, _ in self.pairs]

    @staticmethod
    def _extract(a, t):
        return torch.gather(torch.as_tensor(a, dtype=torch.float), 0, torch.tensor([int(t)]))   # diffusion_utils.py:12-20

    def step_coef(self, t, t_next, eta):
        b = self.b
        bt = self._extract(b, t)
        at = self._extract(self.cumprod, t)
        at_next = torch.ones_like(at) if t_next == -1 else self._extract(self.cumprod, t_next)   # DW:196-199
        c = PixelCoef()
        c.ddpm = 1 if self.sample_type == 'ddpm' else 0
        c.sqrt_at = at.sqrt().item()
        c.sqrt_1m_at = (1 - at).sqrt().item()
        c.sqrt_at_next = at_next.sqrt().item()
        if self.sample_type == 'ddim':
            c1 = eta * ((1 - at / at_next) * (1 - at_next) / (1 - at)).sqrt()                    # DW:217 / 273 / 300
            c2 = ((1 - at_next) - c1 ** 2).sqrt()
            c.c1, c.c2 = c1.item(), c2.item()
        else:
            c.w0 = (at_next.sqrt() * bt / (1 - at)).item()                                        # DW:291
            c.wt = ((1 - bt).sqrt() * (1 - at_next) / (1 - at)).item()                            # DW:292
            c.post_std = (bt * (1 - at_next) / (1 - at)).sqrt().item()                            # DW:295-297
            c.weight = (bt / torch.sqrt(1 - at)).item()                                           # DW:202
            c.inv_sqrt_1m_bt = (1 / torch.sqrt(1.0 - bt)).item()                                  # DW:204
            logvar = self._extract(self.logvar, t)
            c.std_model = torch.exp(0.5 * logvar).item()                                          # DW:208
            c.mask = 1.0 - float(t == 0)                                                          # DW:206
        return c

    def coef_array(self, coefs=None):
        coefs = self.coef if coefs is None else coefs
        return (PixelCoef * len(coefs))(*coefs)
