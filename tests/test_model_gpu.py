"""GPU: model-level parity through the C ABI (t2v_unet_forward / t2v_vae_decode / sampler-step kernels).

Checker = the CPU oracle (oracle/, pinned bit-exact against the reference) and the committed reference outputs in
tests/golden.  The oracle is evaluated in fp32 on the fp16-ROUNDED weights the GPU path holds, so what is measured
is our kernels' arithmetic error, not the weight quantisation.

Tolerances (fp16 storage + fp32 accumulate through ~600 layers): relative RMS error of eps <= RMS_GATE and max |err| <=
MAX_GATE * max|ref| vs the fp32 oracle / reference fixtures = the measured values x 1.5 (DESIGN.md section 5; the gates at
BASELINE's own shapes, with the reference's fp16-autocast path as the yardstick, are in test_parity_gpu.py).
BASELINE.json's element-wise rtol 1e-3 / atol 1e-4 is what the kernel-level tests (test_ops_gpu.py) hold per op."""
import os

import pytest
import torch

from oracle import unet_oracle as UO, vae_oracle as VO, samplers_oracle as SO
from oracle.make_golden import synth_inputs, analytic_model, _SchedModel

from parity_util import report  # noqa: E402

pytestmark = pytest.mark.gpu

RMS_GATE, MAX_GATE = 4e-3, 6e-3      # H100: <= 3.0e-3 / 3.7e-3 over every model-level case (T2V_PARITY_REPORT)


def errs(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).abs().max() / (b.abs().max() + 1e-6)).item(), ((a - b).pow(2).mean().sqrt() / (b.pow(2).mean().sqrt() + 1e-9)).item()


@pytest.fixture(scope='module')
def tiny():
    from t2v_b200.modules import UNetSD
    cfg = UO.UNetConfig(dim=64)
    W = UO.make_weights(UO.param_specs(cfg), seed=1)
    net = UNetSD(dim=64).half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    net.register_schedule(given_betas=SO.linear_sd_betas().numpy())
    Wh = {k: v.half().float() for k, v in W.items()}
    return cfg, W, Wh, net


def test_tiny_unet_vs_reference_fixture_and_taps(tiny, gold_dir):
    cfg, W, Wh, net = tiny
    g = torch.load(os.path.join(gold_dir, 'unet_tiny.pt'))
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    net.enable_taps(True)
    out = net(x.cuda(), torch.tensor([g['t']]).cuda(), c.cuda())
    e = errs(out, g['eps_cond'])
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    for k, v in g.items():
        if k.startswith('tap:'):
            et = errs(net.read_tap(k[4:], tuple(v.shape)), v)
            assert et[1] < RMS_GATE, (k, et)
    net.enable_taps(False)
    out2 = net(x.cuda(), torch.tensor([g['t']]).cuda(), c.cuda())       # arena with buffer reuse
    assert torch.equal(out, out2)
    assert errs(net(x.cuda(), torch.tensor([g['t']]).cuda(), uc.cuda()), g['eps_uncond'])[1] < RMS_GATE


@pytest.mark.parametrize('B,Fr,h,w', [(2, 4, 8, 8), (1, 5, 8, 24), (1, 1, 8, 8), (3, 2, 16, 8)])
def test_tiny_unet_shapes_vs_oracle(tiny, B, Fr, h, w):
    cfg, W, Wh, net = tiny
    g = torch.Generator().manual_seed(B * 100 + Fr)
    x = torch.randn(B, 4, Fr, h, w, generator=g)
    y = torch.randn(B, 77, 1024, generator=g).half().float()
    t = torch.randint(0, 1000, (B,), generator=g)
    ref = UO.unet_forward(Wh, cfg, x, t, y)
    out = net(x.cuda(), t.cuda(), y.cuda())
    e = errs(out, ref)
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    # batched CFG pair == two single forwards (samples are independent: per-sample 5-D GroupNorm / temporal attention)
    if B >= 2:
        single = net(x[:1].cuda(), t[:1].cuda(), y[:1].cuda())
        assert errs(out[:1], single)[1] < 2e-3


def test_float_timesteps_and_longer_context(tiny):
    cfg, W, Wh, net = tiny
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1, 4, 3, 8, 8, generator=g)
    y = torch.randn(1, 154, 1024, generator=g).half().float()         # two 77-token prompt chunks
    t = torch.tensor([437.25])                                          # UniPC passes float times
    ref = UO.unet_forward(Wh, cfg, x, t, y)
    assert errs(net(x.cuda(), t.cuda(), y.cuda()), ref)[1] < RMS_GATE


def test_weight_update_is_picked_up(tiny):
    """LoRA-style re-assignment of a leaf's .weight must invalidate the packed-weight cache."""
    cfg, W, Wh, net = tiny
    g = torch.Generator().manual_seed(4)
    x = torch.randn(1, 4, 2, 8, 8, generator=g).cuda()
    y = torch.randn(1, 77, 1024, generator=g).cuda()
    t = torch.tensor([100]).cuda()
    a = net(x, t, y)
    mod = dict(net.named_modules())['out.2']
    old = mod.weight
    mod.weight = torch.nn.Parameter(old.detach() * 0)
    net.sync_weights(force=True)
    b = net(x, t, y)
    assert not torch.equal(a, b)
    bias = mod.bias.detach().float().view(1, 4, 1, 1, 1)
    assert torch.allclose(b.float(), bias.expand_as(b), atol=1e-3)
    mod.weight = old
    net.sync_weights(force=True)
    assert torch.equal(net(x, t, y), a)


def test_vae_decode_vs_reference_fixture(gold_dir):
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG
    g = torch.load(os.path.join(gold_dir, 'vae_decode.pt'))
    W = UO.make_weights(VO.decoder_param_specs(VO.VAEConfig()), seed=g['wseed'])
    vae = AutoencoderKL(VAE_DDCONFIG, 4).half()
    sd = vae.state_dict()
    sd.update(W)
    vae.load_state_dict(sd, strict=True)
    vae = vae.cuda().eval()
    z = torch.randn(g['z_shape'], generator=torch.Generator('cpu').manual_seed(g['z_seed'])) * g['z_scale']
    out = vae.decode(z.cuda())
    e = errs(out, g['out'])
    report('vae_decode', max=e[0], rms=e[1])
    assert e[1] < 2.1e-3 and e[0] < 2.4e-3, e          # measured 1.38e-3 / 1.57e-3
    # batched video path + fused uint8 conversion == tensor2vid on the float output
    z5 = (z * 0.18215).view(1, 2, 4, 8, 16).permute(0, 2, 1, 3, 4).contiguous()
    u8 = vae.decode_video(z5.cuda(), 1.0 / 0.18215, as_uint8=True).cpu()
    ref_u8 = torch.from_numpy(VO.tensor2vid_u8(g['out'].view(1, 2, 3, 64, 128).permute(0, 2, 1, 3, 4)))
    diff = (u8.int() - ref_u8.int()).abs()
    assert u8.shape == (2, 64, 128, 3) and diff.max() <= 3 and diff.float().mean() < 0.5


@pytest.mark.parametrize('name,key,S,scale', [
    ('DDIM_Gaussian', 'ddim_gaussian_S50_g17.0', 50, 17.0), ('DDIM_Gaussian', 'ddim_gaussian_S7_g1.0', 7, 1.0),
    ('DDIM', 'ddim_S50_g17.0', 50, 17.0), ('DDIM', 'ddim_S20_g7.5', 20, 7.5),
    ('UniPC', 'unipc_S30_g17.0', 30, 17.0), ('UniPC', 'unipc_S12_g7.5', 12, 7.5), ('UniPC', 'unipc_S5_g1.0', 5, 1.0)])
def test_samplers_vs_reference_trajectories(gold_dir, name, key, S, scale):
    """Full trajectories of the three schedulers (fused CUDA step kernels + host coefficient algebra) against the
    reference classes' outputs for the same analytic denoiser.  fp32 throughout -> atol 2e-4."""
    from t2v_b200 import samplers
    g = torch.load(os.path.join(gold_dir, 'samplers.pt'))
    betas = SO.linear_sd_betas()

    class M(_SchedModel):
        def __call__(self, x, t, c):
            return analytic_model(x, t.to(x.device), c)
    model = M(betas)
    model.device = torch.device('cuda')
    x = torch.randn(g['shape'], generator=torch.Generator('cpu').manual_seed(g['x_seed'])).cuda()
    c = torch.full((1, 77, 8), g['c_val']).cuda()
    uc = torch.full((1, 77, 8), g['uc_val']).cuda()
    entry = [s for s in samplers.available_samplers if s.name == name][0]
    smp = entry.init_sampler(model, betas=betas, device=torch.device('cuda'))
    calls = []
    out = smp.sample(S=S, conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=scale, x_T=x,
                     shape=tuple(x.shape), eta=0.0, batch_size=1, callback=lambda *a: calls.append(a))
    assert len(calls) == S
    assert torch.allclose(out.cpu(), g[key], rtol=0, atol=2e-4), (out.cpu() - g[key]).abs().max()


def test_ddim_gaussian_eta_consumes_the_rng_like_the_reference():
    """eta > 0: the reference draws randn_like(xt) for the step noise AND once more in its inpaint hook on every step
    (gaussian_sampler.py:279,:285-291 -- `mask` is overwritten with t.ne(0) at :281, so the hook always runs once attached).
    The oracle restates that; run on the same CUDA generator state the product sampler must give the same latent."""
    from t2v_b200 import samplers
    betas = SO.linear_sd_betas()

    class M(_SchedModel):
        def __call__(self, x, t, c):
            return analytic_model(x, t.to(x.device), c)
    model = M(betas)
    model.device = torch.device('cuda')
    x = torch.randn((1, 4, 5, 6, 7), generator=torch.Generator('cpu').manual_seed(5)).cuda()
    c = torch.full((1, 77, 8), 0.25).cuda()
    uc = torch.full((1, 77, 8), -0.5).cuda()
    smp = samplers.Txt2VideoSampler(model, torch.device('cuda'), betas=betas, sampler_name='DDIM_Gaussian').sampler
    assert hasattr(smp, 'inpaint_masking')
    torch.manual_seed(11)
    out = smp.sample(S=10, conditioning=c, unconditional_conditioning=uc, unconditional_guidance_scale=3.0, x_T=x,
                     shape=tuple(x.shape), eta=0.7, batch_size=1, mask=None)
    torch.manual_seed(11)
    ref = SO.ddim_gaussian_sample(model, betas, x, 10, c, uc, 3.0, eta=0.7)
    assert torch.allclose(out, ref, rtol=0, atol=2e-4), (out - ref).abs().max()


def test_gaussian_cfg_quirk_and_fp16_rounding():
    """DDIM_Gaussian guides channels 0-1 only; CFG is evaluated op by op in fp16 when eps is fp16."""
    from t2v_b200 import _lib
    l = _lib.lib()
    n = 4 * 6
    x = torch.zeros(1, 4, 1, 2, 3, device='cuda')
    ec = torch.ones(1, 4, 1, 2, 3, device='cuda', dtype=torch.half)
    eu = torch.zeros_like(ec)
    out = torch.empty_like(x)
    # x' = a2*x0 + a3*eps with a0 = 1, a1 = 1, a2 = 0, a3 = 1  ->  x' = eps_cfg
    rc = l.t2v_ddim_step(_lib.ptr(x), _lib.ptr(ec), _lib.ptr(eu), 0, _lib.ptr(out), n, 6, 4, 2, 17.0, 0, 1.0, 1.0, 0.0,
                         1.0, 0.0, None, 1, _lib.stream_ptr())
    assert rc == 0
    assert out[0, :, 0, 0, 0].tolist() == [17.0, 17.0, 1.0, 1.0]
    c = torch.randn(n, device='cuda').half()
    u = torch.randn(n, device='cuda').half()
    rc = l.t2v_ddim_step(_lib.ptr(x), _lib.ptr(c), _lib.ptr(u), 0, _lib.ptr(out), n, 6, 4, 4, 7.5, 0, 1.0, 1.0, 0.0, 1.0,
                         0.0, None, 1, _lib.stream_ptr())
    assert rc == 0
    ref = (u + 7.5 * (c - u)).float()          # torch evaluates this in fp16, op by op
    assert torch.equal(out.view(-1), ref)


# ---------------------------------------------------------------------------------------- VideoCrafter (SURVEY.md 8 a19-a20)
from oracle import vc_oracle as VC  # noqa: E402


def _vc_net(cfg, wseed):
    from t2v_b200.modules import UNetModel
    W = UO.make_weights(VC.vc_param_specs(cfg), seed=wseed)
    net = UNetModel(model_channels=cfg.model_channels, context_dim=cfg.context_dim, temporal_length=cfg.temporal_length).half()
    net.load_state_dict(W, strict=True)
    return W, net.cuda().eval()


@pytest.mark.parametrize('name', ['vc_unet_tiny', 'vc_unet_full'])
def test_vc_unet_vs_reference_fixture(gold_dir, name):
    """UNetModel.forward (openaimodel3d.py:632-670) through t2v_unet_forward(arch = 1) vs the reference's fp32 output."""
    g = torch.load(os.path.join(gold_dir, name + '.pt'))
    cfg = VC.VCConfig(**g['cfg'])
    W, net = _vc_net(cfg, g['wseed'])
    B = g['shape'][0]
    x = torch.randn(g['shape'], generator=torch.Generator('cpu').manual_seed(g['x_seed']))
    ctx = torch.randn((B, g['L'], cfg.context_dim), generator=torch.Generator('cpu').manual_seed(g['ctx_seed']))
    out = net(x.cuda(), g['t'].cuda(), context=ctx.cuda())
    e = errs(out, g['out'])
    report('vc:' + name, max=e[0], rms=e[1])
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    assert torch.equal(out, net(x.cuda(), g['t'].cuda(), context=ctx.cuda()))      # graph replay, bit-reproducible


@pytest.mark.parametrize('B,T,h,w', [(1, 4, 8, 16), (2, 3, 16, 8), (1, 5, 8, 8), (1, 9, 8, 8), (1, 24, 8, 8)])
def test_vc_unet_shapes_vs_oracle(B, T, h, w):
    # T > temporal_length + 1 = 5: relative positions clamp to the end rows of the tables (attention_temporal.py:60)
    cfg = VC.VCConfig(model_channels=64, context_dim=48, temporal_length=4)
    W, net = _vc_net(cfg, 5)
    Wh = {k: v.half().float() for k, v in W.items()}
    g = torch.Generator().manual_seed(B * 10 + T)
    x = torch.randn(B, 4, T, h, w, generator=g)
    ctx = torch.randn(B, 9, 48, generator=g).half().float()
    t = torch.randint(0, 1000, (B,), generator=g)
    ref = VC.vc_unet_forward(Wh, cfg, x, t, ctx)
    e = errs(net(x.cuda(), t.cuda(), context=ctx.cuda()), ref)
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e


# ---------------------------------------------------------------------------------------- full-size regressions
def test_full_modelscope_unet_vs_reference_fixture(gold_dir):
    """The public 1.41 B-parameter configuration at BASELINE config 1 (4 frames x 128^2): reference fp32 output."""
    from t2v_b200.modules import UNetSD
    g = torch.load(os.path.join(gold_dir, 'unet_cfg1.pt'))
    cfg = UO.UNetConfig()
    W = UO.make_weights(UO.param_specs(cfg), seed=g['wseed'])
    net = UNetSD().half()
    net.load_state_dict(W, strict=True)
    net = net.cuda().eval()
    x, c, uc = synth_inputs(g['F'], g['h'], g['w'])
    t = torch.tensor([g['t']]).cuda()
    e = errs(net(x.cuda(), t, c.cuda()), g['eps_cond'])
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    assert errs(net(x.cuda(), t, uc.cuda()), g['eps_uncond'])[1] < RMS_GATE


def test_activation_arena_reuse_does_not_change_results(monkeypatch):
    """Regression: the split-K fix-up pass once read partial sums of splits the GEMM never ran (stale arena bytes), which
    only showed at shapes whose K-tile count is not a multiple of the requested split.  The forward must be bit-identical
    with and without activation-buffer reuse."""
    from t2v_b200.modules import UNetSD
    from t2v_b200.synthetic import randomize_
    with torch.device('cuda'):
        net = UNetSD()
    net = randomize_(net.half().cuda().eval(), seed=0)
    for (B, Fr, h, w) in ((1, 4, 16, 16), (2, 3, 8, 24)):
        x = torch.randn(B, 4, Fr, h, w, device='cuda')
        y = torch.randn(B, 77, 1024, device='cuda')
        t = torch.full((B,), 500.0, device='cuda')
        outs = []
        for no_reuse in (True, False):
            if no_reuse:
                monkeypatch.setenv('T2V_ARENA_NO_REUSE', '1')
            else:
                monkeypatch.delenv('T2V_ARENA_NO_REUSE', raising=False)
            p = getattr(net.time_embed, '0').bias
            p.data = p.data.clone()             # re-shipped parameter -> new weights version -> the plan is rebuilt
            net.mark_dirty()
            outs.append(net(x, t, y).clone())
        assert torch.equal(outs[0], outs[1])


# ---------------------------------------------------------------------------------------- VAE encode (vid2vid preparation)
def test_vae_encode_vs_reference_fixture_and_compute_latents(gold_dir):
    """AutoencoderKL.encode(x).mean (t2v_model.py:1640-1644) through t2v_vae_encode vs the reference's fp32 output, and
    compute_latents (t2v_pipeline.py:148-194) on top of it."""
    from t2v_b200.modules import AutoencoderKL
    from t2v_b200.pipeline import VAE_DDCONFIG, TextToVideoSynthesis, SCALE_FACTOR
    g = torch.load(os.path.join(gold_dir, 'vae_encode.pt'))
    cfg = VO.VAEConfig()
    W = {**UO.make_weights(VO.decoder_param_specs(cfg), seed=3), **UO.make_weights(VO.encoder_param_specs(cfg), seed=g['wseed'])}
    ae = AutoencoderKL(VAE_DDCONFIG, 4, None).half()
    ae.load_state_dict(W, strict=True)
    ae = ae.cuda().eval()
    x = torch.rand(g['x_shape'], generator=torch.Generator('cpu').manual_seed(g['x_seed'])) * 2 - 1
    post = ae.encode(x.cuda())
    e = errs(post.mean, g['mean'])
    report('vae_encode_mean', max=e[0], rms=e[1])
    assert e[1] < RMS_GATE and e[0] < MAX_GATE, e
    assert errs(post.logvar, g['logvar'])[1] < 2e-2
    assert post.sample(torch.zeros_like(post.mean)).equal(post.mode())
    # frames with odd tile counts + fp32 input, vs the oracle on the fp16-rounded weights
    Wh = {k: v.half().float() for k, v in W.items()}
    x2 = torch.rand((3, 3, 40, 64), generator=torch.Generator('cpu').manual_seed(9)) * 2 - 1      # mid attention needs h*w % 8 == 0
    ref = VO.vae_encode_moments(Wh, cfg, x2)
    assert errs(ae.encode(x2.cuda()).parameters, ref)[1] < 1e-2
    with pytest.raises(RuntimeError):
        ae.encode(torch.zeros(1, 3, 36, 64).cuda())                      # H not a multiple of 8
    # decode(encode(x)) runs end to end (round trip through both plans)
    rec = ae.decode(post.mode())
    assert rec.shape == (2, 3, 64, 96) and torch.isfinite(rec).all()


# ---------------------------------------------------------------------------------------- LoRA hot-merge (SURVEY.md 8 f4)
def test_lora_hot_merge_matches_reference_arithmetic_and_unmerges_bit_exactly(tiny):
    """StableLoraProcessor.process_lora (stable_lora/stable_utils/lora_processor.py:50-96, :202-246) on the library's packed
    weights: Linear inside the fused q|k|v + LayerNorm-folded copy, the GEGLU projection, a 3x3 conv (tap-major pack), a
    temporal Conv3d (product averaged over the second kernel axis) and a 1x1 projection.  Gate: the hot-merged forward equals
    the forward of a second module whose weights were merged with torch (the reference's ops, fp16) and shipped normally;
    lora_clear() gives back the pre-merge output bit for bit without rebuilding the plan."""
    from t2v_b200.modules import UNetSD
    from t2v_b200.lora import StableLoraProcessor
    cfg, W, Wh, net = tiny
    g = torch.Generator().manual_seed(21)
    x = torch.randn(2, 4, 3, 8, 8, generator=g).cuda()
    y = torch.randn(2, 77, 1024, generator=g).cuda()
    t = torch.tensor([400, 30]).cuda()
    before = net(x, t, y).clone()
    launches = net.num_launches()
    names = ['input_blocks.1.1.transformer_blocks.0.attn1.to_q', 'input_blocks.1.1.transformer_blocks.0.attn2.to_k',
             'input_blocks.1.1.transformer_blocks.0.ff.net.0.proj', 'input_blocks.1.0.in_layers.2',
             'input_blocks.1.0.temopral_conv.conv1.2', 'input_blocks.1.1.proj_in', 'middle_block.1.proj_out']
    mods = dict(net.named_modules())
    rank, alpha = 4, 0.75
    lora, merged_w = {}, {}
    for n in names:
        w = mods[n].weight.detach()
        out_c = w.shape[0]
        cols = w.numel() // out_c
        temporal = w.dim() == 5
        A = (torch.randn(rank, cols * 3 if temporal else cols, generator=g) * 0.2).half().cuda()
        B = (torch.randn(out_c, rank, generator=g) * 0.2).half().cuda()
        lora[n + '.lora_A'], lora[n + '.lora_B'] = A, B
        prod = (B @ A)                                                       # fp16 matmul, fp32 accumulate: autocast's B @ A
        if temporal:
            prod = prod.view(out_c, w.shape[1], 3, 3, 1).mean(dim=-2, keepdim=True)
        merged_w[n + '.weight'] = (w.half() + prod.view(w.shape).half() * alpha)      # process_lora_weight (:50-58), fp16
    n_merged = StableLoraProcessor().process_lora(net, [lora], lora_alpha=alpha)
    assert n_merged == len(names) and net.lora_merged() == len(names)
    hot = net(x, t, y).clone()
    assert not torch.equal(hot, before)
    assert net.num_launches() == launches                                    # same plan, same graph
    # checker: the fp32 oracle on the torch-merged weights (a 1-ulp difference in one merged weight re-rolls the fp16 rounding
    # noise of the whole net -- 2e-3 -- so two fp16 forwards cannot be compared more tightly than each against the oracle)
    sd = {k: v.half().float() for k, v in W.items()}
    for k, v in merged_w.items():
        sd[k] = v.float().cpu()
    orc = UO.unet_forward(sd, cfg, x.cpu(), t.cpu(), y.cpu().half().float())
    e_hot, e_before = errs(hot, orc), errs(before, orc)
    ref_net = UNetSD(dim=64).half()
    ref_net.load_state_dict(sd, strict=True)
    ref_net = ref_net.cuda().eval()
    e_ref = errs(ref_net(x, t, y), orc)                                      # the same merged weights shipped the ordinary way
    report('lora_hot_merge', hot_vs_oracle_rms=e_hot[1], shipped_vs_oracle_rms=e_ref[1], unmerged_vs_oracle_rms=e_before[1])
    assert e_hot[1] < RMS_GATE and e_hot[1] < 1.5 * e_ref[1] + 5e-4, (e_hot, e_ref)
    assert e_before[1] > 10 * e_hot[1], (e_before, e_hot)                    # the merge really changed the function
    # a second merge accumulates on top of the first, like two LoRA files
    net.lora_merge(names[0] + '.weight', lora[names[0] + '.lora_A'], lora[names[0] + '.lora_B'], 0.5)
    assert not torch.equal(net(x, t, y), hot)
    StableLoraProcessor().process_lora(net, [], undo_merge=True)
    assert net.lora_merged() == 0
    assert torch.equal(net(x, t, y), before)                                 # bit-identical to never merging
