"""CPU fp32 restatement of the DiffEdit edit mask (cdx_edit_map / cdx_edit_mask; test infrastructure only).

Per image b and map k: x_t = sqrt_a * x0[b] + sqrt_1ma * noise[b, k] (q_sample's op order), the U-Net on [x_t, x_t] at timestep t
under [c_src[b], c_tgt[b]], d = e_tgt - e_src (times vscale for v nets), s = sum over c ascending of |d|, acc[b] += s with k
ascending.  Then per image: map = acc / (n * C), mean in float64 cast to fp32, M = ratio * mean, mask = min(map, M) / M > 0.5 when
M > 0, else all zeros.  Every op a separate fp32 torch op.
"""
import torch


def q_sample(x0, noise, sqrt_a, sqrt_1ma):
    sa, s1 = torch.tensor(sqrt_a, dtype=torch.float32), torch.tensor(sqrt_1ma, dtype=torch.float32)
    return sa * x0 + s1 * noise


def channel_abs_sum(d):
    """[C, h, w] -> [h, w], |d| summed over c ascending in fp32."""
    s = torch.zeros(d.shape[1:], dtype=torch.float32)
    for c in range(d.shape[0]):
        s = s + d[c].abs()
    return s


def accumulate(e_src, e_tgt, vscale=1.0):
    """[B, n, C, h, w] predictions -> acc [B, h, w], maps added in order."""
    B, n, _, h, w = e_src.shape
    v = torch.tensor(vscale, dtype=torch.float32)
    acc = torch.zeros(B, h, w, dtype=torch.float32)
    for b in range(B):
        for k in range(n):
            acc[b] = acc[b] + channel_abs_sum(v * (e_tgt[b, k] - e_src[b, k]))
    return acc


def edit_map(unet_fn, x0, c_src, c_tgt, t, sqrt_a, sqrt_1ma, noise, vscale=1.0):
    """unet_fn(x [R,C,h,w], t [R] long, c [R,L,D]) -> [R,C,h,w].  noise [B, n, C, h, w] -> acc [B, h, w]."""
    B, n = noise.shape[:2]
    e_src, e_tgt = torch.empty_like(noise), torch.empty_like(noise)
    ts = torch.full((2,), int(t), dtype=torch.long)
    for b in range(B):
        for k in range(n):
            xt = q_sample(x0[b], noise[b, k], sqrt_a, sqrt_1ma)
            e = unet_fn(torch.stack([xt, xt]), ts, torch.stack([c_src[b], c_tgt[b]]))
            e_src[b, k], e_tgt[b, k] = e[0], e[1]
    return accumulate(e_src, e_tgt, vscale)


def normalized(acc, n, C, ratio=3.0):
    """-> (map [B,1,h,w], m / M [B,1,h,w] with m = min(map, M), M [B]) as the mask kernel forms them (M == 0: zeros)."""
    B, h, w = acc.shape
    emap = (acc / torch.tensor(float(n * C), dtype=torch.float32)).unsqueeze(1)
    mean = (emap.double().sum(dim=(1, 2, 3)) / (h * w)).float()
    M = torch.tensor(ratio, dtype=torch.float32) * mean
    Mb = M.view(B, 1, 1, 1)
    norm = torch.where(Mb > 0, torch.minimum(emap, Mb) / torch.where(Mb > 0, Mb, torch.ones_like(Mb)), torch.zeros_like(emap))
    return emap, norm, M


def edit_mask(acc, n, C, ratio=3.0, f=None):
    """-> (map [B,1,h,w], mask [B,1,h,w] in {0, 1}, mask nearest-upsampled by f [B,1,f*h,f*w] or None)."""
    emap, norm, _ = normalized(acc, n, C, ratio)
    mask = (norm > 0.5).float()
    img = None if f is None else mask.repeat_interleave(f, dim=2).repeat_interleave(f, dim=3)
    return emap, mask, img
