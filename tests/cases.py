"""Shared model configurations for the parity tests (small enough for the CPU oracle to finish in seconds)."""
import numpy as np

import oracle

# BASELINE.json configs[0]: the numerics gate (C1).
C1 = dict(kind="vit", image_size=224, patch_size=16, num_classes=1000, dim=192, depth=1, heads=3, mlp_dim=768)

SMALL = {
    "vit_c1": C1,
    "vit_small": dict(kind="vit", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16),
    "vit_mean_rect": dict(kind="vit", image_size=(48, 64), patch_size=(8, 16), num_classes=7, dim=64, depth=1, heads=2,
                          mlp_dim=96, dim_head=32, pool="mean"),
    # widths that are multiples of neither 64 nor 8: every general (non-wgmma, unaligned) kernel path of the bf16 engine
    "vit_odd_dims": dict(kind="vit", image_size=(40, 56), patch_size=8, num_classes=11, dim=50, depth=2, heads=3, mlp_dim=70,
                         dim_head=14, pool="mean"),
    "vit_noproj": dict(kind="vit", image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=1, mlp_dim=64, dim_head=64),
    "deepvit_small": dict(kind="deepvit", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16),
    "cait_small": dict(kind="cait", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, cls_depth=2, heads=4,
                       mlp_dim=128, dim_head=16),
    "crossvit_small": dict(kind="crossvit", image_size=64, num_classes=10, sm_dim=64, lg_dim=128, sm_patch_size=8,
                           lg_patch_size=16, sm_enc_depth=1, lg_enc_depth=2, sm_enc_heads=2, lg_enc_heads=2,
                           sm_enc_mlp_dim=64, lg_enc_mlp_dim=128, sm_enc_dim_head=32, lg_enc_dim_head=32,
                           cross_attn_depth=2, cross_attn_heads=2, cross_attn_dim_head=32, depth=2),
    "parallel_small": dict(kind="parallel_vit", image_size=64, patch_size=16, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128,
                           dim_head=16),
    "parallel_three_noproj": dict(kind="parallel_vit", image_size=32, patch_size=8, num_classes=5, dim=64, depth=2, heads=1,
                                  mlp_dim=64, dim_head=64, num_parallel_branches=3, pool="mean"),
    "merger_small": dict(kind="patch_merger_vit", image_size=64, patch_size=8, num_classes=10, dim=64, depth=4, heads=4, mlp_dim=128,
                         dim_head=16, patch_merge_layer=2, patch_merge_num_tokens=5),
    "merger_default_noproj": dict(kind="patch_merger_vit", image_size=(32, 48), patch_size=8, num_classes=6, dim=64, depth=2, heads=1,
                                  mlp_dim=96, dim_head=64),
    "t2t_small": dict(kind="t2t_vit", image_size=32, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16,
                      t2t_layers=((3, 2), (3, 2))),
    "t2t_default_layers": dict(kind="t2t_vit", image_size=64, num_classes=7, dim=64, depth=1, heads=2, mlp_dim=64, dim_head=32,
                               pool="mean"),
    "crossvit_samedim": dict(kind="crossvit", image_size=32, num_classes=6, sm_dim=64, lg_dim=64, sm_patch_size=8,
                             lg_patch_size=16, sm_enc_depth=1, lg_enc_depth=1, sm_enc_heads=2, lg_enc_heads=2,
                             sm_enc_mlp_dim=64, lg_enc_mlp_dim=64, sm_enc_dim_head=32, lg_enc_dim_head=32,
                             cross_attn_depth=1, cross_attn_heads=2, cross_attn_dim_head=32, depth=1),
}

# Mid-size bf16 cases exercising the tensor-core kernels at the real head / sequence geometry (n = 197, dh = 64).
MID = {
    "vit_mid": dict(kind="vit", image_size=224, patch_size=16, num_classes=1000, dim=256, depth=2, heads=4, mlp_dim=512),
    "parallel_mid": dict(kind="parallel_vit", image_size=224, patch_size=16, num_classes=100, dim=256, depth=2, heads=4, mlp_dim=512),
    "deepvit_mid": dict(kind="deepvit", image_size=224, patch_size=16, num_classes=100, dim=256, depth=2, heads=4, mlp_dim=512),
    "merger_mid": dict(kind="patch_merger_vit", image_size=224, patch_size=16, num_classes=100, dim=256, depth=4, heads=4, mlp_dim=512,
                       patch_merge_layer=2),
    "t2t_mid": dict(kind="t2t_vit", image_size=224, num_classes=100, dim=256, depth=2, heads=4, mlp_dim=512),
    # t2t_small's widths at 288^2 with the default t2t_layers: the first soft-split layer attends over 72^2 = 5184 > 4096 tokens
    # (the three-pass row softmax, kernels.cu softmax_rows_bf16_big_kernel)
    "t2t_big_image": dict(kind="t2t_vit", image_size=288, num_classes=10, dim=64, depth=2, heads=4, mlp_dim=128, dim_head=16),
    "cait_mid": dict(kind="cait", image_size=224, patch_size=16, num_classes=100, dim=192, depth=2, cls_depth=2, heads=4,
                     mlp_dim=384, dim_head=48),
    # dim_head > 64 (ViT-H/14 has 80; 128 is a common setting): plain softmax through scores_mma / mid_fused / pv_mma
    "vit_dh80_p14": dict(kind="vit", image_size=224, patch_size=14, num_classes=100, dim=192, depth=1, heads=4, mlp_dim=256,
                         dim_head=80),
    "vit_dh128": dict(kind="vit", image_size=224, patch_size=16, num_classes=100, dim=192, depth=2, heads=2, mlp_dim=256,
                      dim_head=128),
    # 384^2: 577 tokens, past the rows path's 256 keys, so 8 and 16 heads take mid_fused; CaiT's class layers attn_cls at 578 keys
    "deepvit_384_h8": dict(kind="deepvit", image_size=384, patch_size=16, num_classes=100, dim=128, depth=1, heads=8, mlp_dim=256,
                           dim_head=32),
    "deepvit_384_h16": dict(kind="deepvit", image_size=384, patch_size=16, num_classes=100, dim=128, depth=1, heads=16, mlp_dim=256,
                            dim_head=16),
    "cait_384_h8": dict(kind="cait", image_size=384, patch_size=16, num_classes=100, dim=128, depth=1, cls_depth=1, heads=8,
                        mlp_dim=256, dim_head=32),
    "cait_384_h16": dict(kind="cait", image_size=384, patch_size=16, num_classes=100, dim=128, depth=1, cls_depth=1, heads=16,
                         mlp_dim=256, dim_head=16),
    # the class layers reach attn_cls at dim_head 128
    "cait_dh128": dict(kind="cait", image_size=224, patch_size=16, num_classes=100, dim=192, depth=1, cls_depth=2, heads=2,
                       mlp_dim=256, dim_head=128),
}

# BASELINE.json configs[1..4] (batch replaced by 2: the path has no cross-image op, see test_batch_independence)
FULL = {
    "c2_vit_b16_224": dict(kind="vit", image_size=224, patch_size=16, num_classes=1000, dim=768, depth=12, heads=12, mlp_dim=3072),
    "c3_deepvit_1024x24": dict(kind="deepvit", image_size=224, patch_size=16, num_classes=1000, dim=1024, depth=24, heads=16,
                               mlp_dim=4096),
    "c4_cait_s36_dh48": dict(kind="cait", image_size=224, patch_size=16, num_classes=1000, dim=384, depth=36, cls_depth=2, heads=8,
                             mlp_dim=1536, dim_head=48),
    "c4_cait_s36_dh64": dict(kind="cait", image_size=224, patch_size=16, num_classes=1000, dim=384, depth=36, cls_depth=2, heads=8,
                             mlp_dim=1536, dim_head=64),
    "c5_vit_l16_384": dict(kind="vit", image_size=384, patch_size=16, num_classes=1000, dim=1024, depth=24, heads=16, mlp_dim=4096),
}

# The reference README's usage examples of the two hot-path model classes BASELINE.json has no configuration for (CrossViT: SURVEY.md 8
# a14, README.md:327-345; T2TViT: 8 f3, README.md:208-216), at their own size, batch 2 -- the configurations bench.py --config
# crossvit_readme / t2t_readme time.
README = {
    "crossvit_readme": dict(kind="crossvit", image_size=256, num_classes=1000, depth=4, sm_dim=192, sm_patch_size=16, sm_enc_depth=2,
                            sm_enc_heads=8, sm_enc_mlp_dim=2048, lg_dim=384, lg_patch_size=64, lg_enc_depth=3, lg_enc_heads=8,
                            lg_enc_mlp_dim=2048, cross_attn_depth=2, cross_attn_heads=8),
    "t2t_readme": dict(kind="t2t_vit", image_size=224, num_classes=1000, dim=512, depth=5, heads=8, mlp_dim=512,
                       t2t_layers=((7, 4), (3, 2), (3, 2))),
}


def cfg_of(name):
    d = dict({**SMALL, **MID}[name])
    return oracle.make_config(d.pop("kind"), **d)


def bf16_round(x):
    x = np.ascontiguousarray(x, np.float32)
    u = x.view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)
