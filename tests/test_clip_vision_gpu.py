"""humanvid_b200.CLIPVisionModelWithProjection on an H100, against transformers' CLIPVisionModelWithProjection.

Operators: the spatial attention at head dim 64 against fp32 SDPA, the GEMM's quick-GELU epilogue against fp64 with the guarded-output harness
of test_gemm_paths_gpu.py, and the patchify op against F.unfold.  Network: ViT-L/14 @ 224 and a small config (hidden 256, 4 heads, 2 layers,
patch 32 -> 50 tokens), each with the default random init, with q_proj / k_proj scaled up (peaked attention) and with a few hidden channels
offset ~100x the others' spread.  The native encoder must be no further from transformers in fp32 (TF32 off) than transformers in fp16 eager
(SDPA) is.  Weights are random, rounded to fp16 so every arm sees the same values.  Also: batch independence, determinism, CUDA-graph
replay, errors instead of faults, launch counts and profile categories, and Pose2VideoPipeline with the native encoder."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

transformers = pytest.importorskip("transformers")

pytestmark = pytest.mark.gpu

from conftest import report

if torch.cuda.is_available():
    import humanvid_b200 as hv
    from humanvid_b200._native import ACT_QUICK_GELU, Epilogue, check, i32, i64, lib, ptr, stream
    from test_gemm_paths_gpu import Guarded, bits, check_close, check_inputs_unchanged, cols_mask, gemm_plan, m_for_bst, m_for_ring, rand, sms, strided

def rel(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


@pytest.fixture
def exact_fp32():
    """The fp32 oracle runs in true fp32 (no TF32 convolutions / matmuls)."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


# ------------------------------------------------------------------------------------------------ operators
@pytest.mark.parametrize("qk_scale", [1.0, 8.0])
@pytest.mark.parametrize("NF", [1, 3])
@pytest.mark.parametrize("L", [1, 17, 50, 127, 128, 129, 257, 577])
def test_attention_d64_op(L, NF, qk_scale):
    heads, d, dv = 16, 64, 80
    hp = heads * d
    g = torch.Generator(device="cuda").manual_seed(L * 10 + NF)
    qk = (torch.randn(NF * L, 2 * hp, generator=g, device="cuda") * qk_scale).half()   # [Q | K] per token, as the biased GEMM writes them
    v = torch.randn(NF, L, heads, d, generator=g, device="cuda").half()
    Lp = (L + 7) // 8 * 8
    # V^T as hv_op_gemm_batched_b writes it: rows h*dv .. h*dv+63 = V of head h, row h*dv+64 = ones, rows up to (h+1)*dv zero; the pad
    # columns [L, Lp) of every frame hold the row bias (0 or 1)
    vt = torch.zeros(heads * dv, NF * Lp, device="cuda", dtype=torch.float16)
    for h in range(heads):
        vt[h * dv + d] = 1
        for n in range(NF):
            vt[h * dv : h * dv + d, n * Lp : n * Lp + L] = v[n, :, h].t()
    out = torch.full((NF * L, hp), float("nan"), device="cuda", dtype=torch.float16)
    check(lib().hv_op_attention(ptr(qk), C.c_void_p(qk.data_ptr() + 2 * hp), ptr(vt), ptr(out), i64(NF), i64(L), i32(heads), i32(d), i64(2 * hp),
                                i64(2 * hp), i64(NF * Lp), i64(hp), None, None, i64(0), i64(0), i64(0), i64(1), i64(0), i64(Lp), i64(0), stream()))
    q = qk[:, :hp].float().view(NF, L, heads, d).transpose(1, 2)
    k = qk[:, hp:].float().view(NF, L, heads, d).transpose(1, 2)
    ref = F.scaled_dot_product_attention(q, k, v.float().transpose(1, 2)).transpose(1, 2).reshape(NF * L, hp)
    e = rel(out, ref)
    report(f"attention d64 op heads={heads} NF={NF} L={L} qk x{qk_scale:g}: rel vs fp32 SDPA {e:.2e}")
    assert torch.isfinite(out).all() and e <= 1e-3


@pytest.mark.parametrize("d", [24, 48, 56, 96, 128])
def test_attention_rejects_head_dims_without_instantiation(d):
    x = torch.zeros(128, 4096, device="cuda", dtype=torch.float16)
    assert lib().hv_op_attention(ptr(x), ptr(x), ptr(x), ptr(x), i64(1), i64(64), i32(2), i32(d), i64(4096), i64(4096), i64(4096), i64(4096),
                                 None, None, i64(0), i64(0), i64(0), i64(1), i64(0), i64(64), i64(0), stream()) != 0


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


# name: (M rule, N, K, residual, want BLOCK_N, want BST).  M rule: an int, or "ring" / "bst" (derived from the SM count as in
# test_gemm_paths_gpu.py).  The encoder's fc1 runs at M = 257 B, N = 4096, K = 1024.
QG = {
    "fc1_b1": (257, 4096, 1024, False, None, False),
    "fc1_b2_res": (514, 4096, 1024, True, None, False),
    "ring128_partial_n": ("ring", 328, 1000, False, 128, False),
    "ring128_partial_n_res": ("ring", 328, 1000, True, 128, False),
    "ring256_res": ("ring", 1280, 1280, True, 256, False),
    "bst128": ("bst", 384, 320, False, 128, True),
    "bst128_partial_n_res": ("bst", 328, 200, True, 128, True),
    "bst256_partial_n": ("bst", 488, 200, False, 256, True),
}


@pytest.mark.parametrize("name", list(QG))
def test_gemm_quick_gelu(name):
    mrule, N, K, with_res, want_bn, want_bst = QG[name]
    s = sms()
    if mrule == "bst":
        M = m_for_bst((N + want_bn - 1) // want_bn, s)
    elif mrule == "ring":
        M = m_for_ring(N, want_bn, s)
    else:
        M = mrule
    bn, stages, grid = gemm_plan(M, N, K)
    plan = f"{name}: M={M} N={N} K={K} -> BLOCK_N {bn}, {'BST ' + str(stages) + ' stages' if stages else 'ring'}, grid {grid}"
    report("quick-GELU gemm plan " + plan)
    if want_bn is not None:
        assert bn == want_bn, plan
    assert (stages > 0) == want_bst, plan
    A = strided(M, K, K + 16, seed=1)
    W = rand(N, K, scale=K ** -0.5, seed=3)
    bias = rand(N, seed=4)
    inputs = [A, W, bias]
    ref = quick_gelu(A.double() @ W.double().t() + bias.double())
    ep = Epilogue(bias=bias.data_ptr(), act=ACT_QUICK_GELU)
    if with_res:
        res = strided(M, N, N + 40, seed=6)
        ep.residual, ep.ldr = res.data_ptr(), N + 40
        inputs.append(res)
        ref = ref + res.double()
    ldc = N + 24
    before = [bits(t) for t in inputs]
    g = Guarded(M, ldc)
    check(lib().hv_op_gemm(ptr(A), i64(A.stride(0)), None, i64(0), i64(0), ptr(W), ptr(g.out), i64(ldc), i64(M), i64(N), i64(K), C.byref(ep), stream()))
    torch.cuda.synchronize()
    g.check_untouched(cols_mask(M, ldc, N), name)
    check_inputs_unchanged(before, inputs, name)
    e = check_close(g.out[:, :N], ref, name, block_n=bn)
    report(f"quick-GELU gemm {name}: rel vs fp64 {e:.2e}")


@pytest.mark.parametrize("B, S, p, Kpad", [(1, 224, 14, 640), (3, 224, 32, 3072), (2, 56, 14, 592)])
def test_patchify_op(B, S, p, Kpad):
    x = torch.randn(B, 3, S, S, device="cuda").half()
    g = S // p
    out = torch.full((B * g * g, Kpad), float("nan"), device="cuda", dtype=torch.float16)
    check(lib().hv_op_clip_patchify(ptr(x), ptr(out), i64(B), i64(3), i64(S), i64(p), i64(Kpad), stream()))
    torch.cuda.synchronize()
    ref = F.unfold(x, kernel_size=p, stride=p).transpose(1, 2).reshape(B * g * g, 3 * p * p)   # (c, ky, kx) order = the conv weight's
    assert torch.equal(bits(out[:, : 3 * p * p]), bits(ref))
    assert torch.equal(bits(out[:, 3 * p * p :]), torch.zeros_like(bits(out[:, 3 * p * p :])))


def test_patchify_rejects_bad_shapes():
    x = torch.zeros(1, 3, 224, 224, device="cuda", dtype=torch.float16)
    out = torch.zeros(256, 640, device="cuda", dtype=torch.float16)
    assert lib().hv_op_clip_patchify(ptr(x), ptr(out), i64(1), i64(3), i64(224), i64(15), i64(680), stream()) == -1   # 224 % 15
    assert lib().hv_op_clip_patchify(ptr(x), ptr(out), i64(1), i64(3), i64(224), i64(14), i64(584), stream()) == -1   # Kpad < 588
    assert lib().hv_op_clip_patchify(ptr(x), ptr(out), i64(1), i64(3), i64(224), i64(14), i64(596), stream()) == -1   # Kpad % 8


# ------------------------------------------------------------------------------------------------ network
CONFIGS = {
    "small": dict(hidden_size=256, intermediate_size=1024, projection_dim=64, num_hidden_layers=2, num_attention_heads=4, image_size=224, patch_size=32),
    "vit_l14": dict(hidden_size=1024, intermediate_size=4096, projection_dim=768, num_hidden_layers=24, num_attention_heads=16, image_size=224,
                    patch_size=14),
}


def make_hf(cfg_name, variant):
    """transformers' model (eager attention) with random weights rounded to fp16 (kept in fp32)."""
    torch.manual_seed(1234)
    cfg = transformers.CLIPVisionConfig(**CONFIGS[cfg_name], attn_implementation="eager")
    m = transformers.CLIPVisionModelWithProjection(cfg).eval()
    sd = {k: v.half().float() for k, v in m.state_dict().items()}
    C_ = cfg.hidden_size
    if variant == "qk_scaled":
        # q and k rows of std 2 / sqrt(hidden): scores of std ~4 per head, so attention is far from uniform
        for k in sd:
            if k.endswith(("q_proj.weight", "k_proj.weight")):
                sd[k] = (sd[k] * (2.0 / C_ ** 0.5) / sd[k].std()).half().float()
    elif variant == "offsets":
        # a few residual-stream channels carry offsets ~100x the spread of the others (pre_layrnorm output has unit spread per row)
        for ch, off in ((3, 100.0), (77, -100.0), (150, 60.0), (200, -80.0)):
            sd["vision_model.pre_layrnorm.bias"][ch] = off
    m.load_state_dict(sd)
    return m, sd


@pytest.fixture(scope="module")
def arms_cache():
    return {}


def arms(cache, cfg_name, variant):
    key = (cfg_name, variant)
    if key not in cache:
        cache.clear()
        torch.cuda.empty_cache()
        m32, sd = make_hf(cfg_name, variant)
        m32 = m32.cuda()
        m16 = transformers.CLIPVisionModelWithProjection(transformers.CLIPVisionConfig(**CONFIGS[cfg_name], attn_implementation="sdpa")).eval()
        m16.load_state_dict(sd)
        m16 = m16.half().cuda()
        nat = hv.CLIPVisionModelWithProjection(**CONFIGS[cfg_name])
        nat.load_state_dict(sd)
        nat = nat.to("cuda", torch.float16)
        cache[key] = (m32, m16, nat)
    return cache[key]


def pixels(B, S, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(B, 3, S, S, generator=g, device="cuda") * 1.2).half()


@pytest.mark.parametrize("variant", ["default", "qk_scaled", "offsets"])
@pytest.mark.parametrize("cfg_name", ["small", "vit_l14"])
def test_parity_vs_transformers(arms_cache, exact_fp32, cfg_name, variant):
    m32, m16, nat = arms(arms_cache, cfg_name, variant)
    B = 2
    pix = pixels(B, 224, 11)
    with torch.no_grad():
        o32 = m32(pix.float(), output_attentions=variant == "qk_scaled")
        o16 = m16(pix)
        on = nat(pix)
    torch.cuda.synchronize()
    L = (224 // CONFIGS[cfg_name]["patch_size"]) ** 2 + 1
    assert on.image_embeds.shape == (B, CONFIGS[cfg_name]["projection_dim"]) and on.image_embeds.dtype == torch.float16
    assert on.last_hidden_state.shape == (B, L, CONFIGS[cfg_name]["hidden_size"])
    assert torch.isfinite(on.image_embeds).all() and torch.isfinite(on.last_hidden_state).all()
    e_emb, e_emb16 = rel(on.image_embeds, o32.image_embeds), rel(o16.image_embeds, o32.image_embeds)
    e_hid, e_hid16 = rel(on.last_hidden_state, o32.last_hidden_state), rel(o16.last_hidden_state, o32.last_hidden_state)
    extra = ""
    if variant == "qk_scaled":
        rowmax = torch.cat([a.amax(-1).flatten() for a in o32.attentions])
        med = float(rowmax.median())
        extra = f"; median row-max attention probability {med:.3f} (uniform: {1 / L:.3f})"
        assert med > 10.0 / L
    report(f"clip {cfg_name} {variant} B={B}: image_embeds native vs fp32 {e_emb:.2e}, fp16-eager vs fp32 {e_emb16:.2e}; last_hidden_state "
           f"native {e_hid:.2e}, fp16-eager {e_hid16:.2e}{extra}")
    assert e_hid <= e_hid16
    if variant == "offsets":
        # Both arms hold the residual stream in fp16, where the offset channels sit at |x| ~ 100 (spacing 0.0625) and dominate the
        # post_layernorm statistics of the class token; which way those roundings fall decides image_embeds.  Measured on an H100: for the
        # same two ViT-L images, transformers fp16's own error is 1.85e-3 in a batch of 2 and 1.98e-3 in a batch of 16 (the native
        # encoder's is 1.99e-3 in both), and over 16 images the per-image errors of the two arms agree to 3 digits on 14 of them.
        assert e_emb <= 1.1 * e_emb16
    else:
        assert e_emb <= e_emb16


def test_batch_independence_determinism_graph(arms_cache):
    _, _, nat = arms(arms_cache, "vit_l14", "default")
    pix = pixels(3, 224, 5)
    with torch.no_grad():
        a = nat(pix)
        b = nat(pix)
        assert torch.equal(a.image_embeds, b.image_embeds) and torch.equal(a.last_hidden_state, b.last_hidden_state)
        for i in range(3):
            s = nat(pix[i : i + 1])
            assert torch.equal(s.image_embeds[0], a.image_embeds[i]), i
            assert torch.equal(s.last_hidden_state[0], a.last_hidden_state[i]), i
        emb_t, hid_t = nat(pix, return_dict=False)
        assert torch.equal(emb_t, a.image_embeds) and torch.equal(hid_t, a.last_hidden_state)
        # CUDA graph: the forward never allocates or synchronises once the workspace is reserved
        h = nat._sync_native()
        nat.reserve_workspace(3)
        ps = pix.clone()
        emb = torch.empty_like(a.image_embeds)
        hid = torch.empty_like(a.last_hidden_state)
        fwd = lambda: check(lib().hv_clip_vision_forward(h, ptr(ps), ptr(emb), ptr(hid), i32(3), None, C.c_size_t(0), stream()), h)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            fwd()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            fwd()
        ps.copy_(pixels(3, 224, 6))
        graph.replay()
        torch.cuda.synchronize()
        c = nat(ps)
        assert torch.equal(emb, c.image_embeds) and torch.equal(hid, c.last_hidden_state)
        ps.copy_(pix)
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(emb, a.image_embeds) and torch.equal(hid, a.last_hidden_state)
        # without last_hidden_state the embeddings are the same
        emb2 = torch.empty_like(emb)
        check(lib().hv_clip_vision_forward(h, ptr(pix), ptr(emb2), None, i32(3), None, C.c_size_t(0), stream()), h)
        torch.cuda.synchronize()
        assert torch.equal(emb2, a.image_embeds)
        # launch count and profile categories: patchify, patch GEMM, embeddings LN, 8 per layer, class-token copy, post LN, projection
        nat(pix)
        layers = CONFIGS["vit_l14"]["num_hidden_layers"]
        assert nat.last_launch_count == 8 * layers + 6
        check(lib().hv_set_profiling(h, i32(1)), h)
        nat(pix)
        ms, fl = (C.c_double * 6)(), (C.c_double * 6)()
        cnt = (C.c_int64 * 6)()
        check(lib().hv_get_profile(h, ms, fl, cnt, i32(6)), h)
        check(lib().hv_set_profiling(h, i32(0)), h)
    assert cnt[0] == 5 * layers + 1 and cnt[2] == layers and cnt[4] == 2 * layers + 2 and cnt[5] == 1 and cnt[1] == 0 and cnt[3] == 0
    assert fl[2] == layers * 4.0 * 257 * 257 * 1024 * 3 and ms[2] > 0


def test_errors_not_faults(arms_cache):
    _, _, nat = arms(arms_cache, "small", "default")
    with pytest.raises(ValueError):
        nat(torch.zeros(1, 3, 256, 256, device="cuda", dtype=torch.float16))
    h = nat._sync_native()
    f = lib().hv_workspace_bytes
    f.restype = C.c_size_t
    assert f(h, i32(1), i32(1), i32(200), i32(200)) == 0
    assert lib().hv_reserve_workspace(h, i32(1), i32(1), i32(256), i32(256)) == -1
    assert b"224" in lib().hv_last_error(h)
    need = f(h, i32(2), i32(1), i32(224), i32(224))
    assert need > 0
    pix = pixels(2, 224, 1)
    emb = torch.zeros(2, 64, device="cuda", dtype=torch.float16)
    ws = torch.empty(need // 2, device="cuda", dtype=torch.uint8)
    assert lib().hv_clip_vision_forward(h, ptr(pix), ptr(emb), None, i32(2), ptr(ws), C.c_size_t(need // 2), stream()) == -1
    assert b"workspace too small" in lib().hv_last_error(h)
    assert lib().hv_clip_vision_forward(h, ptr(pix), ptr(emb), None, i32(0), None, C.c_size_t(0), stream()) == -1
    torch.cuda.synchronize()
    # the handle still works
    ws = torch.empty(need, device="cuda", dtype=torch.uint8)
    check(lib().hv_clip_vision_forward(h, ptr(pix), ptr(emb), None, i32(2), ptr(ws), C.c_size_t(need), stream()), h)
    torch.cuda.synchronize()
    assert torch.equal(emb, nat(pix).image_embeds)


# ------------------------------------------------------------------------------------------------ pipeline
MM_KW = dict(num_attention_heads=8, num_transformer_block=1, attention_block_types=["Temporal_Self", "Temporal_Self"],
             temporal_position_encoding=True, temporal_position_encoding_max_len=32, temporal_attention_dim_div=1)


def test_pose2video_pipeline_with_native_image_encoder(arms_cache):
    from humanvid_b200.pipeline import Pose2VideoPipeline, _to_tensor_image
    from oracle import hv_oracle as O
    import vae_oracle as V

    _, _, enc = arms(arms_cache, "small", "default")
    dev = "cuda"
    chs, xdim, Fv, H, W = (64, 128, 256, 256), 64, 24, 128, 128
    assert enc.config.projection_dim == xdim
    unet = hv.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim, use_motion_module=True, use_inflated_groupnorm=True,
                                   motion_module_resolutions=(1, 2, 4, 8), motion_module_mid_block=True, motion_module_type="Vanilla",
                                   motion_module_kwargs=MM_KW, unet_use_cross_frame_attention=False, unet_use_temporal_attention=False)
    unet.load_state_dict(O.synthetic_init(O.UNet3DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=7).half().float().state_dict())
    pg = hv.PoseGuider(64, block_out_channels=(16, 32, 96, 256))
    pg.load_state_dict(O.synthetic_init(O.PoseGuider(64, 3, (16, 32, 96, 256)).eval(), seed=11).half().float().state_dict())
    cam = hv.CameraPoseEncoder(downscale_factor=8, channels=[64], nums_rb=2, cin=384, ksize=1, sk=True, use_conv=False, compression_factor=1,
                               temporal_attention_nhead=8, attention_block_types=["Temporal_Self"], temporal_position_encoding=True,
                               temporal_position_encoding_max_len=24)
    cam.load_state_dict(O.synthetic_init(O.CameraPoseEncoder(channels=(64,), heads=8).eval(), seed=13).half().float().state_dict())
    ref_unet = hv.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim)
    ref_unet.load_state_dict(O.synthetic_init(O.UNet2DConditionModel(block_out_channels=chs, cross_attention_dim=xdim).eval(), seed=17).half().float().state_dict())
    vae = hv.AutoencoderKL()
    vae.load_state_dict(O.synthetic_init(V.AutoencoderKL().eval(), seed=21).half().float().state_dict())
    sched = hv.DDIMScheduler(beta_start=0.00085, beta_end=0.012, beta_schedule="linear", clip_sample=False, steps_offset=1,
                             prediction_type="v_prediction", rescale_betas_zero_snr=True, timestep_spacing="trailing")
    pipe = Pose2VideoPipeline(vae=vae, image_encoder=enc, reference_unet=ref_unet, denoising_unet=unet, pose_guider=pg,
                              camera_pose_encoder=cam, scheduler=sched).to(dev, torch.float16)
    g = torch.Generator(device=dev).manual_seed(3)
    ref = torch.rand(3, H, W, generator=g, device=dev) * 2 - 1
    poses = [torch.rand(1, 3, H, W, generator=g, device=dev) for _ in range(Fv)]
    camera = torch.randn(1, 6, Fv, H, W, generator=g, device=dev).half()
    vid = pipe(ref, poses, camera, W, H, Fv, 1, 3.5, generator=torch.Generator(device=dev).manual_seed(7), output_type="tensor").videos
    vid = torch.as_tensor(vid)
    assert vid.shape == (1, 3, Fv, H, W) and torch.isfinite(vid.float()).all()
    # the pipeline's conditioning is the module's image_embeds of the same pixels
    emb = pipe._clip_embed(ref, dev)
    pix = _to_tensor_image(ref, 224, 224).to(dev) * 0.5 + 0.5
    mean = torch.tensor(pipe.clip_image_processor.image_mean, device=dev).view(1, 3, 1, 1)
    std = torch.tensor(pipe.clip_image_processor.image_std, device=dev).view(1, 3, 1, 1)
    direct = enc(((pix - mean) / std).half()).image_embeds
    assert emb.dtype == torch.float16 and emb.shape == (1, xdim)
    assert torch.equal(emb, direct)
    report(f"pipeline 24 frames 128x128 with native image encoder: image_embeds norm {float(emb.float().norm()):.3f}, video mean {float(vid.float().mean()):.3f}")
