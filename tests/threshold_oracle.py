"""TEST INFRASTRUCTURE ONLY -- CPU fp32 restatement of DDIM_Gaussian's x0 range restriction.

  * `quantile`          torch.quantile(v, q, dim=1) with linear interpolation, as ATen computes it: rank = fp32(q) * (n - 1) in
                        fp32, the floor(rank)-th and ceil(rank)-th order statistics, torch.lerp's fp32 arithmetic (w < 0.5 ?
                        a + w (b - a) : b - (b - a)(1 - w), each op rounded), NaN for a row holding a NaN, and torch's
                        "input tensor is too large" error above 2^24 elements.  This is what the radix select of
                        csrc/quantile.cu must reproduce bit for bit.
  * `restrict_x0`       restrict_range_x0 (gaussian_sampler.py:110-120) as p_mean_variance calls it (:174-178): `percentile`
                        wins; s = max(quantile(|x0|), 1) per sample (the reference runs one sample, where its [B]-shaped s
                        acts as a scalar); otherwise any non-None `clamp` clamps to [-1, 1] (it is called with clamp=True).
  * `threshold_step`    one DDIM_Gaussian update on given eps in the fp32 (and fp16 CFG) op order of t2v_ddim_step_threshold.
  * `ddim_gaussian_sample_restricted`
                        GaussianDiffusion.sample (:214-296) with `clamp` / `percentile`: oracle/samplers_oracle.py's loop with
                        the restriction between mean_x0 and get_eps; `s_trace` collects each step's s.

Pinned by tests/test_ddim_threshold_cpu.py against tests/golden/ddim_threshold.pt, which
scripts/make_golden_ddim_threshold.py writes from the reference's own GaussianDiffusion.
"""
import torch

from oracle import samplers_oracle as SO

QUANTILE_MAX_N = 1 << 24


def quantile(v, q):
    """v [B, n] fp32 -> [B]."""
    if v.numel() > QUANTILE_MAX_N:
        raise RuntimeError('quantile() input tensor is too large')
    n = v.shape[1]
    srt = torch.sort(v, dim=1).values                       # NaN sorts last
    rank = torch.tensor(q, dtype=torch.float32) * (n - 1)   # fp32
    lo, hi = int(torch.floor(rank)), int(torch.ceil(rank))
    w = rank - lo
    a, b = srt[:, lo], srt[:, hi]
    d = b - a
    out = a + w * d if float(w) < 0.5 else b - d * (1 - w)
    return torch.where(torch.isnan(v).any(dim=1), torch.full_like(out, float('nan')), out)


def abs_quantile_rows(x0, q):
    """One s per sample of x0 [B, ...]: quantile(|x0|) row by row, so B > 1 does not trip the 2^24 limit of the whole batch."""
    v = x0.flatten(1).abs()
    return torch.cat([quantile(v[i:i + 1], q) for i in range(v.shape[0])])


def restrict_x0(x0, clamp=None, percentile=None, s_trace=None):
    if percentile is not None:
        assert percentile > 0 and percentile <= 1
        s = abs_quantile_rows(x0, percentile)
        if s_trace is not None:
            s_trace.append(s.clone())
        s = s.clamp(1.0).view(-1, *((1,) * (x0.dim() - 1)))
        return torch.min(s, torch.max(-s, x0)) / s
    if clamp is not None:
        return x0.clamp(-True, True)
    return x0


def threshold_step(x, e_c, e_u, g, guided_channels, coefs, noise, cfg_fp16, clamp=None, percentile=None):
    """x [B, C, ...] fp32, e_c / e_u fp16 or fp32 -> x_{t-1}; coefs = (sr, srm1, sqrt(alpha_prev), direction, mask * sigma)."""
    a0, a1, a2, a3, a4 = (float(c) for c in coefs)
    e = e_c.float().clone()
    if e_u is not None:
        ec, eu = e_c[:, :guided_channels], e_u[:, :guided_channels]
        e[:, :guided_channels] = ((eu + g * (ec - eu)) if cfg_fp16 else (eu.float() + g * (ec.float() - eu.float()))).float()
    ax = a0 * x
    x0 = restrict_x0(ax - a1 * e, clamp, percentile)
    eps = (ax - x0) / a1
    nz = a4 * noise if (noise is not None and a4 != 0.0) else 0.0
    return a2 * x0 + a3 * eps + nz


@torch.no_grad()
def ddim_gaussian_sample_restricted(model, betas, x_T, S, cond, uncond, guide_scale, eta=0.0, clamp=None, percentile=None,
                                    trace=None, s_trace=None):
    acp = torch.cumprod(1 - betas, dim=0)
    sqrt_recip = torch.sqrt(1.0 / acp)
    sqrt_recipm1 = torch.sqrt(1.0 / acp - 1)
    ts, stride = SO.gaussian_timesteps(len(betas), S)
    xt = x_T.clone()
    for step in range(S):
        t = torch.full((xt.shape[0],), int(ts[step]), dtype=torch.long)
        if guide_scale is None or guide_scale == 1:
            out = model(xt, t, cond)
        else:
            out = SO.gaussian_cfg(model(xt, t, cond), model(xt, t, uncond), guide_scale)
        x0 = SO._i(sqrt_recip, t, xt) * xt - SO._i(sqrt_recipm1, t, xt) * out
        x0 = restrict_x0(x0, clamp, percentile, s_trace)
        alphas = SO._i(acp, t, xt)
        alphas_prev = SO._i(acp, (t - stride).clamp(0), xt)
        eps = (SO._i(sqrt_recip, t, xt) * xt - x0) / SO._i(sqrt_recipm1, t, xt)
        sigmas = eta * torch.sqrt(((1 - alphas_prev) / (1 - alphas)) * (1 - alphas / alphas_prev))
        noise = torch.randn_like(xt)
        direction = torch.sqrt(1 - alphas_prev - sigmas ** 2) * eps
        mask = t.ne(0).float().view(-1, *((1,) * (xt.ndim - 1)))
        xt = torch.sqrt(alphas_prev) * x0 + direction + mask * sigmas * noise
        torch.randn_like(xt)     # the inpaint-mask hook's unused draw (:285-291)
        if trace is not None:
            trace.append(xt.clone())
    return xt
