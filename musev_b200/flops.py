"""Algorithmic work of one `UNet3DConditionModel.forward` (the figure the roofline uses; SURVEY.md section 8d).

Counts 2*M*N*K for every conv / linear the REFERENCE executes and 4*BH*Nq*Nk*d for every attention call -- true,
unpadded dimensions; the dead CFG recompute (Q3) and the no-op AdaIN (Q2) are excluded. For the baseline shape
(B=2, T=16+1, 64x64) this reproduces the numbers measured on the reference with hooks: 48.336 TFLOP (`musev`),
54.153 TFLOP (`musev_referencenet`). `vae_encoder_flops` / `vae_decoder_flops` count the two VAE halves the same way
(equal to torch's FlopCounterMode on the oracles, tests/test_vae_encoder_host.py).
"""
from __future__ import annotations

from typing import Dict

from .schema import UNetConfig, refer_emb_shapes


def unet_forward_flops(cfg: UNetConfig, B: int, T: int, H: int, W: int, n_text: int = 77, n_clip: int = 4,
                       n_vis_cond: int = 1, n_ref_frames: int = 1) -> Dict[str, float]:
    f = {"conv": 0.0, "linear": 0.0, "attention": 0.0}
    heads = cfg.heads
    NF = B * T
    temb = cfg.temb_dim
    X = cfg.cross_attention_dim

    def conv(M, cin, cout, taps):
        f["conv"] += 2.0 * M * cout * cin * taps

    def lin(M, K, N):
        f["linear"] += 2.0 * M * N * K

    def attn(bh, nq, nk, d):
        f["attention"] += 4.0 * bh * nq * nk * d

    def tblock_linears(M, C, kv_dim, kv_rows, ip):
        lin(M, C, C)                       # attn1 q
        lin(kv_rows[0], C, C); lin(kv_rows[0], C, C)      # attn1 k, v
        lin(M, C, C)                       # attn1 out
        lin(M, C, C)                       # attn2 q
        lin(kv_rows[1], kv_dim, C); lin(kv_rows[1], kv_dim, C)
        if ip:
            lin(kv_rows[2], kv_dim, C); lin(kv_rows[2], kv_dim, C)
        lin(M, C, C)                       # attn2 out
        lin(M, C, 8 * C); lin(M, 4 * C, C)  # GEGLU ff

    def resnet(hw, cin, C):
        M = NF * hw
        conv(M, cin, C, 9)
        lin(NF, temb, C)
        conv(M, C, C, 9)
        if cin != C:
            conv(M, cin, C, 1)

    def temp_conv(hw, C):
        for _ in range(4):
            conv(NF * hw, C, C, 3)

    def spatial(hw, C):
        M = NF * hw
        d = C // heads
        conv(M, C, C, 1); conv(M, C, C, 1)          # proj_in / proj_out
        n_self = hw + (n_vis_cond * hw if (cfg.need_t2i_ip_adapter and n_vis_cond > 0 and T > 1) else 0)
        # the reference projects K/V of the concatenated (own + vis-cond) tokens for every frame
        tblock_linears(M, C, X, (NF * n_self, NF * n_text, NF * n_clip), cfg.ip_adapter_cross_attn)
        attn(NF * heads, hw, n_self, d)
        attn(NF * heads, hw, n_text, d)
        if cfg.ip_adapter_cross_attn:
            attn(NF * heads, hw, n_clip, d)

    def temporal(hw, C):
        M = NF * hw
        d = C // heads
        lin(M, C, C); lin(M, C, C)                   # proj_in / proj_out
        lin(B * T, temb, C)                          # frame_emb_proj
        tblock_linears(M, C, C, (M, M, 0), False)
        attn(B * hw * heads, T, T, d)
        attn(B * hw * heads, T, T, d)

    def refer(hw, C, nref):
        M = NF * hw
        d = C // heads
        lin(M, C, C)
        lin(NF * (nref + hw), C, C); lin(NF * (nref + hw), C, C)
        lin(M, C, C)
        attn(NF * heads, hw, nref + hw, d)

    boc = cfg.block_out_channels
    nb = len(boc)
    hw = H * W
    conv(NF * hw, cfg.in_channels, boc[0], 9)
    lin(B, boc[0], temb); lin(B, temb, temb)
    lin(B * T, boc[0], temb); lin(B * T, temb, temb)
    if cfg.need_transformer_in:
        temporal(hw, boc[0])
    ref_shapes = None
    if cfg.need_refer_emb:
        ref_shapes, mid_shape = refer_emb_shapes(cfg, H, W)
        refer(hw, boc[0], n_ref_frames * ref_shapes[0][1] * ref_shapes[0][2])
    ch = boc[0]
    h, w = H, W
    for i in range(nb):
        final = i == nb - 1
        cin, ch = ch, boc[i]
        num_block = cfg.layers_per_block + (0 if final else 1)
        start = 1 + num_block * i
        for j in range(cfg.layers_per_block):
            resnet(h * w, cin if j == 0 else ch, ch)
            temp_conv(h * w, ch)
            if not final:
                spatial(h * w, ch)
                temporal(h * w, ch)
            if cfg.need_refer_emb:
                rs = ref_shapes[start + j]
                refer(h * w, ch, n_ref_frames * rs[1] * rs[2])
        if not final:
            h, w = h // 2, w // 2
            conv(NF * h * w, ch, ch, 9)
            if cfg.need_refer_emb:
                rs = ref_shapes[start + cfg.layers_per_block]
                refer(h * w, ch, n_ref_frames * rs[1] * rs[2])
    cm = boc[-1]
    resnet(h * w, cm, cm); temp_conv(h * w, cm); spatial(h * w, cm); temporal(h * w, cm)
    resnet(h * w, cm, cm); temp_conv(h * w, cm)
    if cfg.need_refer_emb:
        refer(h * w, cm, n_ref_frames * mid_shape[1] * mid_shape[2])
    rev = list(reversed(boc))
    ch = rev[0]
    for i in range(nb):
        prev, ch = ch, rev[i]
        cin_block = rev[min(i + 1, nb - 1)]
        for j in range(cfg.layers_per_block + 1):
            skip = cin_block if j == cfg.layers_per_block else ch
            resnet(h * w, (prev if j == 0 else ch) + skip, ch)
            temp_conv(h * w, ch)
            if i > 0:
                spatial(h * w, ch)
                temporal(h * w, ch)
        if i != nb - 1:
            h, w = h * 2, w * 2
            conv(NF * h * w, ch, ch, 9)
    conv(NF * h * w, boc[0], cfg.out_channels, 9)
    f["gemm"] = f["conv"] + f["linear"]
    f["total"] = f["gemm"] + f["attention"]
    return f


def _vae_mid_flops(conv, lin, attn, NF: int, hw: int, cm: int) -> None:
    """UNetMidBlock2D of the VAE: two resnets and one single-head attention of dim cm over the hw tokens of a frame."""
    for _ in range(2):
        conv(NF * hw, cm, cm, 9); conv(NF * hw, cm, cm, 9)
    for _ in range(4):                       # q, k, v, to_out
        lin(NF * hw, cm, cm)
    attn(NF, hw, hw, cm)


def _vae_counters():
    f = {"conv": 0.0, "linear": 0.0, "attention": 0.0}

    def conv(M, cin, cout, taps):
        f["conv"] += 2.0 * M * cout * cin * taps

    def lin(M, K, N):
        f["linear"] += 2.0 * M * N * K

    def attn(bh, nq, nk, d):
        f["attention"] += 4.0 * bh * nq * nk * d

    return f, conv, lin, attn


def _vae_total(f: Dict[str, float]) -> Dict[str, float]:
    f["gemm"] = f["conv"] + f["linear"]
    f["total"] = f["gemm"] + f["attention"]
    return f


def vae_encoder_flops(cfg, N: int, h: int, w: int) -> Dict[str, float]:
    """`AutoencoderKL.encode` of N images of (h * 2^(nb-1)) x (w * 2^(nb-1)) pixels (h, w = latent size; VAEConfig `cfg`):
    Encoder.forward + quant_conv (diffusers models/vae.py:133-175, autoencoder_kl.py:284). SD-1.5 at 64x64 latents
    (one 512x512 image): 1.117 TFLOP."""
    f, conv, lin, attn = _vae_counters()
    boc, nb = cfg.block_out_channels, len(cfg.block_out_channels)
    H, W = h * 2 ** (nb - 1), w * 2 ** (nb - 1)
    conv(N * H * W, cfg.in_channels, boc[0], 9)
    ch = boc[0]
    for i in range(nb):
        prev, ch = ch, boc[i]
        for j in range(cfg.layers_per_block):
            cin = prev if j == 0 else ch
            conv(N * H * W, cin, ch, 9); conv(N * H * W, ch, ch, 9)
            if cin != ch:
                conv(N * H * W, cin, ch, 1)
        if i != nb - 1:
            H, W = H // 2, W // 2
            conv(N * H * W, ch, ch, 9)
    _vae_mid_flops(conv, lin, attn, N, H * W, boc[-1])
    zc2 = 2 * cfg.latent_channels
    conv(N * H * W, boc[-1], zc2, 9)
    conv(N * H * W, zc2, zc2, 1)
    return _vae_total(f)


def vae_decoder_flops(cfg, N: int, h: int, w: int) -> Dict[str, float]:
    """`AutoencoderKL.decode` of N latents of h x w (VAEConfig `cfg`): post_quant_conv + Decoder.forward (diffusers
    models/autoencoder_kl.py:283, models/vae.py:265-316). SD-1.5 at 64x64 latents (one 512x512 image): 2.515 TFLOP."""
    f, conv, lin, attn = _vae_counters()
    boc, nb = cfg.block_out_channels, len(cfg.block_out_channels)
    zc, cm = cfg.latent_channels, boc[-1]
    H, W = h, w
    conv(N * H * W, zc, zc, 1)
    conv(N * H * W, zc, cm, 9)
    _vae_mid_flops(conv, lin, attn, N, H * W, cm)
    ch = cm
    for i in range(nb):
        prev, ch = ch, boc[nb - 1 - i]
        for j in range(cfg.layers_per_block + 1):
            cin = prev if j == 0 else ch
            conv(N * H * W, cin, ch, 9); conv(N * H * W, ch, ch, 9)
            if cin != ch:
                conv(N * H * W, cin, ch, 1)
        if i != nb - 1:
            H, W = H * 2, W * 2
            conv(N * H * W, ch, ch, 9)
    conv(N * H * W, boc[0], cfg.out_channels, 9)
    return _vae_total(f)


def pose_guider_flops(cfg, N: int, H: int, W: int) -> Dict[str, float]:
    """`PoseGuider.forward` on N images of H x W (PoseGuiderConfig `cfg`; musev/models/controlnet.py:361-371), 2 M N K per
    3x3 convolution over the reference's channel counts (padding channels are not counted). (16, 32, 96, 256) -> 320 at
    512 x 512: 14.72 GFLOP per frame."""
    from .schema import pose_guider_layers
    f, conv, _, _ = _vae_counters()
    for _, cin, cout, stride in pose_guider_layers(cfg):
        H, W = (H - 1) // stride + 1, (W - 1) // stride + 1
        conv(N * H * W, cin, cout, 9)
    return _vae_total(f)


def clip_vision_flops(cfg, N: int) -> Dict[str, float]:
    """`CLIPVisionModelWithProjection.forward` on N images (ClipVisionConfig `cfg`; transformers models/clip/modeling_clip.py),
    2 M N K per matrix product: the patch conv, q / k / v / out_proj / fc1 / fc2 per layer, q k^T and P v per head, and
    visual_projection on the class token. ViT-H/14 at 224 x 224: 0.3346 TFLOP per image."""
    f, conv, lin, attn = _vae_counters()
    C, I, T = cfg.hidden_size, cfg.intermediate_size, cfg.num_patches + 1
    conv(N * cfg.num_patches, cfg.num_channels, C, cfg.patch_size ** 2)
    for _ in range(cfg.num_hidden_layers):
        for _ in range(4):                      # q, k, v, out_proj
            lin(N * T, C, C)
        attn(N * cfg.num_attention_heads, T, T, C // cfg.num_attention_heads)
        lin(N * T, C, I)
        lin(N * T, I, C)
    lin(N, C, cfg.projection_dim)
    return _vae_total(f)


def clip_text_flops(cfg, N: int, L: int) -> Dict[str, float]:
    """`CLIPTextModel.forward` on N sequences of L tokens (ClipTextConfig `cfg`; transformers models/clip/modeling_clip.py),
    2 M N K per matrix product: q / k / v / out_proj / fc1 / fc2 per layer, and q k^T and P v per head over all L x L pairs
    (the causal mask is an addend; the reference's eager attention multiplies the masked pairs too). SD-1.5 at L = 77:
    13.30 GFLOP per sequence."""
    f, conv, lin, attn = _vae_counters()
    C, I = cfg.hidden_size, cfg.intermediate_size
    for _ in range(cfg.num_hidden_layers):
        for _ in range(4):                      # q, k, v, out_proj
            lin(N * L, C, C)
        attn(N * cfg.num_attention_heads, L, L, C // cfg.num_attention_heads)
        lin(N * L, C, I)
        lin(N * L, I, C)
    return _vae_total(f)
