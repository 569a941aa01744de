"""fp64 references of the attention kernels' operations, on the same fp16 operands the kernels read, and the per-element
error gate derived from the kernels' numerics (see tests/test_attention_gpu.py for the derivation).

Operands are addressed as the kernels address them: a flat fp16 storage, batch b at (b // b_inner) * bs + (b % b_inner) * bsi,
row s at s * ss, head h at column h * hd.  The reference is chunked over queries so that a 9216-token frame stays a few
hundred MB in fp64."""
import torch

U16 = 2.0 ** -11          # unit roundoff of fp16 (round to nearest)
U32 = 2.0 ** -24          # unit roundoff of fp32
U32T = 2.0 ** -23         # fp32 accumulation inside the tensor cores (allowed to truncate)
SUB16 = 2.0 ** -25        # half the fp16 subnormal spacing: absolute rounding error below 2^-14
TINY16 = 2.0 ** -14       # smallest normal fp16
GATE_K = 2.0              # gate = GATE_K * bound


def flat(t):
    """The 1-D fp16 storage that starts at t's first element (t may be a column slice of a fused matrix)."""
    n = t.untyped_storage().nbytes() // t.element_size() - t.storage_offset()
    return torch.as_strided(t, (n,), (1,), t.storage_offset())


def gather(t, S, heads, hd, bs, ss, bmap, b_inner=1, bsi=0):
    """[len(bmap), S, heads, hd] fp64: for entry i, batch bmap[i] of the operand that starts at t's first element."""
    dev = t.device
    f = flat(t)
    b = bmap.to(dev).long()
    boff = (b // b_inner) * bs + (b % b_inner) * bsi
    off = (boff[:, None, None, None] + torch.arange(S, device=dev)[None, :, None, None] * ss
           + torch.arange(heads, device=dev)[None, None, :, None] * hd + torch.arange(hd, device=dev)[None, None, None, :])
    return f[off].double()


class Ref:
    """out: the fp64 result [B, Sq, H, D].  pv = sum_j p_j |v_j| (values incl. the relative-position rows), pv_tab = the
    table part of it, tiny = sum over the keys with 0 < p_j < 2^-14 of |v_j| (where fp16 P rounding is absolute), sabs =
    max_j sum_d |q_d| |k_jd| and smax = max_j |scale * s_j| per query row ([B, Sq, H, 1])."""

    def __init__(self, out, pv, pv_tab, tiny, sabs, smax):
        self.out, self.pv, self.pv_tab, self.tiny, self.sabs, self.smax = out, pv, pv_tab, tiny, sabs, smax


def attention64(q, k, v, scale, *, causal=False, rk=None, rv=None, max_rel=0, chunk=1024):
    """softmax(scale * (q k^T [+ q Rk[clamp(s - t, -L, L) + L]^T])) (v [+ Rv[...]]) in fp64; causal: keys s <= t only.
    q [B, Sq, H, D], k / v [B, Skv, H, D] (fp64, K / V already expanded to q's batches); rk / rv [>= 2L+1, D]."""
    dev = q.device
    qh, kh, vh = (x.permute(0, 2, 1, 3) for x in (q, k, v))          # [B, H, S, D]
    Sq, Skv = qh.shape[2], kh.shape[2]
    kt, kta, va = kh.transpose(-1, -2), kh.abs().transpose(-1, -2), vh.abs()
    res = {n: [] for n in ('out', 'pv', 'pv_tab', 'tiny', 'sabs', 'smax')}
    j = torch.arange(Skv, device=dev)
    for c0 in range(0, Sq, chunk):
        qc = qh[:, :, c0:c0 + chunk]
        t = torch.arange(c0, c0 + qc.shape[2], device=dev)
        s = qc @ kt
        sa = qc.abs() @ kta
        if rk is not None:
            idx = (j[None, :] - t[:, None]).clamp(-max_rel, max_rel) + max_rel          # [n, Skv]
            rki, rvi = rk.double()[idx], rv.double()[idx]                              # [n, Skv, D]
            s = s + torch.einsum('bhtd,tsd->bhts', qc, rki)
            sa = sa + torch.einsum('bhtd,tsd->bhts', qc.abs(), rki.abs())
        s = s * scale
        valid = (j[None, :] <= t[:, None]) if causal else torch.ones(len(t), Skv, dtype=torch.bool, device=dev)
        s = s.masked_fill(~valid, float('-inf'))
        p = torch.softmax(s, dim=-1)
        tinym = ((p > 0) & (p < TINY16)).double()
        out, pv, tiny = p @ vh, p @ va, tinym @ va
        pv_tab = torch.zeros_like(pv)
        if rk is not None:
            out = out + torch.einsum('bhts,tsd->bhtd', p, rvi)
            pv_tab = torch.einsum('bhts,tsd->bhtd', p, rvi.abs())
            pv = pv + pv_tab
            tiny = tiny + torch.einsum('bhts,tsd->bhtd', tinym, rvi.abs())
        res['out'].append(out)
        res['pv'].append(pv)
        res['pv_tab'].append(pv_tab)
        res['tiny'].append(tiny)
        res['sabs'].append(sa.masked_fill(~valid, 0).amax(-1, keepdim=True))
        res['smax'].append(s.abs().masked_fill(~valid, 0).amax(-1, keepdim=True))
    return Ref(*(torch.cat(res[n], dim=2).permute(0, 2, 1, 3) for n in ('out', 'pv', 'pv_tab', 'tiny', 'sabs', 'smax')))


def gate(r, *, hd, scale, n_acc, n_l, p_round=True, tab_round=False, exact_scores=False):
    """GATE_K x the error bound of one output element (module docstring of tests/test_attention_gpu.py)."""
    E = 0.0 if exact_scores else scale * hd * U32T * r.sabs + 2 * U32T * r.smax + 2 * U32T
    bound = ((U16 + n_l * U32) * r.out.abs() + SUB16 + E * (r.pv + r.out.abs())
             + (p_round * U16 + n_acc * U32T) * r.pv + SUB16 * r.tiny)
    if tab_round:
        bound = bound + U16 * r.pv_tab
    return GATE_K * bound


def flash_counts(skv, tile):
    """(n_acc, n_l) of the online-softmax kernels: P.V adds one fp32 rounding per 16-key MMA step plus two per tile
    (rescale), a thread sums its skv / 4 probabilities of a row sequentially, then 2 shuffles, the rescales and 1 / l."""
    n_tiles = -(-skv // tile)
    return skv / 16 + 2 * n_tiles + 4, skv / 4 + 2 * n_tiles + 4
