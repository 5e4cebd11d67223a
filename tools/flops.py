"""Algorithmic FLOP / byte counts of the hot path (roofline numerators; multiply-add = 2).  SURVEY.md §8(d) / BASELINE.md §3.
Product-side restatement for bench.py and the measurement tools (the oracle keeps its own copy; tests assert they agree)."""


def dit_block_flops(cfg, L, Lc=512):
    d, ffn = cfg["dim"], cfg["ffn_dim"]
    blk = 8 * L * d * d + 4 * L * L * d + (4 * L * d * d + 4 * Lc * d * d + 4 * L * Lc * d) + 4 * L * d * ffn
    if cfg["has_image_input"]:
        blk += 4 * 257 * d * d + 4 * L * 257 * d
    return blk


def dit_forward_flops(cfg, L, Lc=512):
    d = cfg["dim"]
    pre = 2 * L * (4 * cfg["in_dim"]) * d + 2 * Lc * cfg["text_dim"] * d + 2 * Lc * d * d + 2 * L * d * 64
    return cfg["num_layers"] * dit_block_flops(cfg, L, Lc) + pre


def self_attention_flops(cfg, Lq, Lk):
    return 4.0 * Lq * Lk * cfg["dim"]


def vae_decode_flops(t_lat, h, w):
    """h, w: latent size.  (0.688 + 2.162 (T_lat - 1)) GFLOP per latent position."""
    return (0.688 + 2.162 * (t_lat - 1)) * 1e9 * h * w


def vae_encode_flops(t_lat, H, W):
    """H, W: pixel size.  (6.66 + 5.00 (T_lat - 1)) MFLOP per pixel position."""
    return (6.66 + 5.00 * (t_lat - 1)) * 1e6 * H * W


def vae_min_bytes(t_lat, h, w):
    """Minimal conv in+out traffic (bf16) of the VAE decoder per clip: 8.5 GB per latent frame at 480p (60x104), SURVEY §8d."""
    return 8.5e9 * t_lat * (h * w) / 6240.0


def rife_interp_flops(H, W, scale=1.0):
    """Algorithmic FLOPs of one interpolated frame (RIFE IFNet, 3 blocks x 2 directions; torch.utils.flop_counter's count
    on the reference module): 102.4 GFLOP at 832x480, 236.3 GFLOP at 1280x720 (scale 1)."""
    tot = 0.0
    for s in (4 / scale, 2 / scale, 1 / scale):
        p2, p4 = (H / s) * (W / s) / 4, (H / s) * (W / s) / 16
        macs = p2 * 45 * 11 * 9 + p4 * 90 * 45 * 9 + 8 * p4 * 90 * 90 * 9 + 2 * p4 * 90 * 45 * 16 + p2 * 45 * (4 + 1) * 16
        tot += 2 * 2 * macs
    return tot


def esrgan_flops(H, W):
    """Algorithmic FLOPs of one ESRGAN x4 frame (RRDBNet, 23 blocks, 64 features, growth 32) from an H x W input:
    35.85 MFLOP per input pixel, 14.3 TFLOP at 832x480 and 33.0 TFLOP at 1280x720."""
    k = 9                                                             # 3x3 taps
    rdb = k * 32 * (64 + 96 + 128 + 160) + k * 192 * 64              # conv1..4 (growth) + conv5
    macs = (k * 3 * 64 + 23 * 3 * rdb + k * 64 * 64                  # conv_first, body, conv_body at 1x
            + 4 * k * 64 * 64                                         # conv_up1 at 2x
            + 16 * (2 * k * 64 * 64 + k * 64 * 3))                    # conv_up2, conv_hr, conv_last at 4x
    return 2.0 * macs * H * W
