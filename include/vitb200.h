/* libvitb200 -- C-ABI of the H100-native ViT-family forward engine.
 *
 * The reference (taki0112/vit-tensorflow) has NO plugin / FFI interface: its hot path sits behind plain
 * Python classes (SURVEY.md section 8b).  The boundary preserved is the constructor + call surface
 *     ViT(...)(img) -> logits        vit_tensorflow/vit.py:107-108,159-177
 *     DeepViT(...)(img)              vit_tensorflow/deepvit.py:113-114,139-157
 *     CaiT(...)(img)                 vit_tensorflow/cait.py:156-157,180-194
 *     CrossViT(...)(img)             vit_tensorflow/cross_vit.py:233-253,290-303
 *     parallel_vit.ViT(...)(img)     vit_tensorflow/parallel_vit.py:120-133,167-185   (SURVEY.md 8f, f3)
 *     T2TViT(...)(img)               vit_tensorflow/t2t.py:50-54,96-116               (SURVEY.md 8f, f3)
 *     vit_with_patch_merger.ViT(...)(img)   vit_tensorflow/vit_with_patch_merger.py:134-146,174-185   (8f, f4)
 *     efficient.ViT(...)(img)        vit_tensorflow/efficient.py:13-14,39-55 = vb_forward_embed -> caller's transformer -> vb_forward_head
 *     LeViT(...)(img)                vit_tensorflow/levit.py:164-226 (vb_create_levit; distillation head: vb_forward_distill)
 *     CvT(...)(img)                  vit_tensorflow/cvt.py:149-202 (vb_create_cvt)
 *     TwinsSVT(...)(img)             vit_tensorflow/twins_svt.py:215-268 (vb_create_twins_svt)
 *     CrossFormer(...)(img)          vit_tensorflow/crossformer.py:205-269 (vb_create_crossformer)
 *     NesT(...)(img)                 vit_tensorflow/nest.py:150-216 (vb_create_nest)
 *     RegionViT(...)(img)            vit_tensorflow/regionvit.py:184-263 (vb_create_regionvit)
 *     ScalableViT(...)(img)          vit_tensorflow/scalable_vit.py:250-319 (vb_create_scalable_vit)
 *     PiT(...)(img)                  vit_tensorflow/pit.py:158-219 (vb_create_pit)
 *     MAE(...)(img) / SimMIM(...)(img)   vit_tensorflow/mae.py:49-92, simmim.py:82-129 (vb_create_mim, vb_forward_mim)
 *     MPP(...)(img)                      vit_tensorflow/mpp.py:168-218 (vb_create_mim, vb_forward_mpp)
 *     DistillWrapper(...)([img, labels])  vit_tensorflow/distill.py:87-134 (vb_create_distill, vb_forward_distill_loss)
 * and this header is what the Python host classes (vit_tensorflow_b200/models.py, _lib.py) bind with ctypes.
 * Plain pointers and sizes only; no torch / C++ types cross the boundary.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; the message is vb_last_error(handle)
 *     (pass NULL for errors of vb_create / the vb_op_* helpers).  Nothing throws or aborts across the ABI.
 *   - a handle is bound to one CUDA device and is not thread-safe; distinct handles are independent.
 *   - weights: caller keeps ownership of host arrays, the engine copies/packs them to the device.
 *   - images are NHWC float32 (vit.py:159, usage vit.py:193), logits float32 [batch, num_classes].
 */
#ifndef VITB200_H_
#define VITB200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VB_ABI_VERSION 7
#if defined(__GNUC__)
#define VB_API __attribute__((visibility("default")))
#else
#define VB_API
#endif

typedef struct vb_handle vb_handle;

enum { VB_KIND_VIT = 0, VB_KIND_DEEPVIT = 1, VB_KIND_CAIT = 2, VB_KIND_CROSSVIT = 3, VB_KIND_PARALLEL_VIT = 4,
       VB_KIND_PATCH_MERGER_VIT = 5, VB_KIND_T2T_VIT = 6, VB_KIND_CCT = 7, VB_KIND_LEVIT = 8,
       VB_KIND_CVT = 9, VB_KIND_TWINS_SVT = 10, VB_KIND_CROSSFORMER = 11, VB_KIND_NEST = 12, VB_KIND_REGIONVIT = 13,
       VB_KIND_ATS_VIT = 14, VB_KIND_SMALL_DATASET_VIT = 15, VB_KIND_MOBILEVIT = 16,
       VB_KIND_SCALABLE_VIT = 17, VB_KIND_PIT = 18, VB_KIND_MAE = 19, VB_KIND_SIMMIM = 20, VB_KIND_MPP = 21 };
enum { VB_CCT_POS_SINE = 0, VB_CCT_POS_LEARNABLE = 1, VB_CCT_POS_NONE = 2 };   /* cct.py:233-234,250-256 */
enum { VB_PRECISION_FP32 = 0, VB_PRECISION_BF16 = 1 };
enum { VB_POOL_CLS = 0, VB_POOL_MEAN = 1 };
enum { VB_MEM_HOST = 0, VB_MEM_DEVICE = 1 };

/* Constructor kwargs of the reference classes, flattened.  Unused fields are ignored per kind. */
typedef struct vb_config {
  int32_t struct_size;            /* sizeof(vb_config), ABI guard */
  int32_t kind;                   /* VB_KIND_* */
  int32_t precision;              /* VB_PRECISION_*: FP32 = exact-fp32 SIMT path (numerics gate); BF16 = tensor-core path */
  int32_t image_h, image_w;       /* vit.py:133 pair(image_size) */
  int32_t patch_h, patch_w;       /* vit.py:134 pair(patch_size) */
  int32_t channels;               /* 3 */
  int32_t num_classes;
  int32_t dim, depth, heads, dim_head, mlp_dim;
  int32_t pool;                   /* VB_POOL_* (vit.py:139,170-173) */
  int32_t cls_depth;              /* CaiT (cait.py:156) */
  int32_t max_batch;              /* workspace is sized for this batch */
  /* CrossViT (cross_vit.py:233-253) */
  int32_t sm_dim, lg_dim;
  int32_t sm_patch_size, sm_enc_depth, sm_enc_heads, sm_enc_mlp_dim, sm_enc_dim_head;
  int32_t lg_patch_size, lg_enc_depth, lg_enc_heads, lg_enc_mlp_dim, lg_enc_dim_head;
  int32_t cross_attn_depth, cross_attn_heads, cross_attn_dim_head;
  int32_t cross_depth;            /* CrossViT `depth`: number of multi-scale blocks */
  int32_t parallel_branches;      /* parallel ViT `num_parallel_branches` (parallel_vit.py:130); ignored by the other kinds */
  /* vit_with_patch_merger.ViT (vit_with_patch_merger.py:104-109,141-142) */
  int32_t patch_merge_layer_index;   /* default(patch_merge_layer, depth // 2) - 1: merge AFTER this layer; outside [0, depth) = never */
  int32_t patch_merge_num_tokens;
  /* T2TViT `t2t_layers` (t2t.py:54): up to 4 (kernel_size, stride) soft-split layers; image_h == image_w, patch_* unused */
  int32_t t2t_num_layers;
  int32_t t2t_k0, t2t_s0, t2t_k1, t2t_s1, t2t_k2, t2t_s2, t2t_k3, t2t_s3;
  /* CCT (cct.py:307-339; appended within ABI 7): a Tokenizer of cct_conv_layers x [Conv2D(cct_kernel, cct_stride, SAME,
   * no bias) -> ReLU -> MaxPool2D(cct_pool_kernel, cct_pool_stride, SAME)], 64 channels between layers and `dim` after the last;
   * cct_pos_emb: VB_CCT_POS_*.  Uses dim, depth, heads, dim_head (= dim / heads), mlp_dim, num_classes, image_h / image_w. */
  int32_t cct_conv_layers, cct_kernel, cct_stride, cct_pool_kernel, cct_pool_stride, cct_pos_emb;
} vb_config;

/* A client built against the ABI-7 struct before the CCT fields were appended passes struct_size = VB_CONFIG_SIZE_ABI7;
 * vb_create reads only that prefix and treats the fields after it as zero. */
#define VB_CONFIG_SIZE_ABI7 ((int32_t)(45 * sizeof(int32_t)))

VB_API int vb_abi_version(void);

/* Replaces <Model>.__init__ (vit.py:107-157 etc.): validates the config and allocates device state.  VB_KIND_LEVIT, VB_KIND_CVT,
 * VB_KIND_TWINS_SVT, VB_KIND_CROSSFORMER, VB_KIND_NEST and VB_KIND_REGIONVIT are refused here: their handles come from
 * vb_create_levit, vb_create_cvt, vb_create_twins_svt, vb_create_crossformer, vb_create_nest and vb_create_regionvit (and the
 * other extension kinds from their own vb_create_*; VB_KIND_MAE, VB_KIND_SIMMIM and VB_KIND_MPP from vb_create_mim). */
VB_API int vb_create(const vb_config* cfg, int device, vb_handle** out);

/* LeViT (levit.py:164-212), appended within ABI 7.  `dims`, `depths` and `heads` hold `stages` entries each (cast_tuple already
 * applied, :180-182).  The stem is four Conv2D(3x3, stride 2, SAME, bias) going channels -> 32 -> 64 -> 128 -> dims[0]; stage s
 * is depths[s] x (Attention(dims[s], heads[s], dim_key, dim_value) + MLP(mlp_mult)) on a fmap x fmap map (fmap = image_h / 16,
 * halved with ceil after each shrink); between stages s and s+1 one shrink block: attention with 2 * heads[s] heads whose queries
 * are the even pixels, to dims[s+1], then an MLP of multiplier 2 (:203).  Head: global average pool -> Dense(num_classes), plus
 * Dense(num_distill_classes) when num_distill_classes > 0 (:210). */
#define VB_LEVIT_MAX_STAGES 8
typedef struct vb_levit_config {
  int32_t struct_size;            /* sizeof(vb_levit_config) */
  int32_t stages;                 /* 1 .. VB_LEVIT_MAX_STAGES */
  int32_t dims[VB_LEVIT_MAX_STAGES], depths[VB_LEVIT_MAX_STAGES], heads[VB_LEVIT_MAX_STAGES];
  int32_t dim_key, dim_value, mlp_mult;
  int32_t num_distill_classes;    /* 0: no distillation head */
} vb_levit_config;

/* LeViT.__init__: `base` supplies precision, image_h == image_w (image_size, a multiple of 16), channels, num_classes and
 * max_batch; its kind must be VB_KIND_LEVIT and its other fields are ignored.  Weights (SURVEY.md App. B) are named by the
 * reference's attribute paths: conv_embedding.{i}.kernel [3, 3, cin, cout] / .bias, backbone.{t}.layers.{l}.0.{to_q,to_k,to_v}.0
 * .kernel [1, 1, cin, cout] with the BatchNormalization .1.{gamma,beta,moving_mean,moving_variance}, .0.pos_bias.embeddings
 * [fmap^2, heads], .0.to_out.1.kernel / .bias and .0.to_out.2.{BatchNormalization}, .1.net.0 / .1.net.3 .kernel / .bias (the
 * MLP), mlp_head and distill_head .kernel / .bias.  vb_finalize folds every BatchNormalization (inference statistics, eps 1e-5)
 * into its convolution. */
VB_API int vb_create_levit(const vb_config* base, const vb_levit_config* lv, int device, vb_handle** out);

/* CvT (cvt.py:149-202), appended within ABI 7: the reference's three stages s1, s2, s3 (index 0, 1, 2).  Stage s is a
 * Conv2D(emb_dim, emb_kernel, emb_stride, SAME, bias) over the previous map, the channel LayerNorm (eps 1e-5, cvt.py:30-43), then
 * depth x [x = attn(LN(x)) + x; x = mlp(LN(x)) + x] with heads of 64 (dim_head is fixed, cvt.py:130,189): q = pw_q(BN(dw_q(y))),
 * kv = pw_kv(BN(dw_kv(y))) with depthwise proj_kernel x proj_kernel SAME convolutions of stride 1 and kv_proj_stride (no bias),
 * softmax(q k^T / 8) v, to_out (1x1, bias); mlp = 1x1 (emb_dim * mlp_mult, bias) -> exact GELU -> 1x1 (emb_dim, bias).  Head:
 * GlobalAvgPool2D -> Dense(num_classes).  No position embeddings: any image size. */
#define VB_CVT_STAGES 3
typedef struct vb_cvt_config {
  int32_t struct_size;            /* sizeof(vb_cvt_config) */
  int32_t emb_dim[VB_CVT_STAGES], emb_kernel[VB_CVT_STAGES], emb_stride[VB_CVT_STAGES];
  int32_t proj_kernel[VB_CVT_STAGES];      /* 1 .. 7 */
  int32_t kv_proj_stride[VB_CVT_STAGES];   /* 1 or 2 */
  int32_t heads[VB_CVT_STAGES], depth[VB_CVT_STAGES], mlp_mult[VB_CVT_STAGES];
} vb_cvt_config;

/* CvT.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_CVT and its other
 * fields (image size included: CvT takes any h x w at call time) are ignored.  Weights (SURVEY.md App. B) are named by the
 * reference's attribute paths: cvt_layers.{s}.0.kernel [k, k, cin, emb_dim] / .bias, cvt_layers.{s}.1.g / .b [1, 1, 1, emb_dim],
 * cvt_layers.{s}.2.layers.{l}.0.norm.g / .b, ....0.fn.to_q.net.0.kernel [k, k, 1, emb_dim] (depthwise), .net.1.{gamma, beta,
 * moving_mean, moving_variance}, .net.2.kernel [1, 1, emb_dim, 64 * heads], the same for to_kv with 128 * heads,
 * ....0.fn.to_out.0.kernel / .bias, ....1.norm.g / .b, ....1.fn.net.0 / .net.3 .kernel / .bias, cvt_layers.3.1.kernel / .bias
 * (the Dense head).  vb_finalize folds every BatchNormalization (inference statistics, eps 1e-5) into the depthwise taps and a
 * per-channel shift. */
VB_API int vb_create_cvt(const vb_config* base, const vb_cvt_config* cvt, int device, vb_handle** out);

/* Twins-SVT (twins_svt.py:215-268), appended within ABI 7: the reference's four stages s1 .. s4 (index 0 .. 3).  Stage s is
 * PatchEmbedding ('b (h p1) (w p2) c -> b h w (c p1 p2)', then a 1x1 Conv2D with bias), Transformer(depth 1), PEG (x + a
 * depthwise peg_kernel_size SAME Conv2D with bias), Transformer(depth[s]).  A Transformer layer is x = x + f(LN(x)) for f = local
 * attention within local_patch_size windows, MLP, global attention against the keys of a Conv2D(global_k, stride global_k, VALID),
 * MLP; stage 4 has no local attention and no first MLP (has_local=False, :255).  Every stage has 8 heads of 64 and an MLP
 * multiplier of 4 (Transformer is never passed them, :254-258); the LayerNorm is the module's own (eps 1e-5, :45-58).  Head:
 * GlobalAvgPool2D -> Dense(num_classes).  No position embeddings: any image whose maps are divisible by each patch_size and, in
 * stages 1-3, local_patch_size, and are at least global_k on each side. */
#define VB_TWINS_STAGES 4
typedef struct vb_twins_svt_config {
  int32_t struct_size;            /* sizeof(vb_twins_svt_config) */
  int32_t emb_dim[VB_TWINS_STAGES], patch_size[VB_TWINS_STAGES], local_patch_size[VB_TWINS_STAGES], global_k[VB_TWINS_STAGES];
  int32_t depth[VB_TWINS_STAGES];
  int32_t peg_kernel_size;        /* 1 .. 7 */
} vb_twins_svt_config;

/* TwinsSVT.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_TWINS_SVT and its
 * other fields are ignored.  Weights (SURVEY.md App. B) are named by the reference's attribute paths, for stage s and layer l:
 * svt_layers.{s}.0.proj.kernel [1, 1, cin * p^2, emb_dim] / .bias (the c-slowest patch vector), svt_layers.{s}.{1|3}.layers.{l}.{0|1|2|3}
 * .fn.norm.g / .b [1, 1, 1, emb_dim] (0 local attention, 1 and 3 MLPs, 2 global attention), ....0.fn.fn.to_q.kernel [1, 1, emb_dim,
 * 512], ....0.fn.fn.to_kv.kernel [1, 1, emb_dim, 1024], ....{0|2}.fn.fn.to_out.0.kernel [1, 1, 512, emb_dim] / .bias,
 * ....{1|3}.fn.fn.net.0.kernel [1, 1, emb_dim, 4 emb_dim] / .bias, ....net.3.kernel / .bias, ....2.fn.fn.to_q.kernel,
 * ....2.fn.fn.to_kv.kernel [global_k, global_k, emb_dim, 1024], svt_layers.{s}.2.proj.fn.kernel [k, k, 1, emb_dim] / .bias (PEG),
 * svt_layers.4.1.kernel / .bias (the Dense head).  Stage 4 has no .0 / .1 sub-blocks. */
VB_API int vb_create_twins_svt(const vb_config* base, const vb_twins_svt_config* tw, int device, vb_handle** out);

/* CrossFormer (crossformer.py:205-269), appended within ABI 7: four stages, each a CrossEmbedLayer (:30-48: one SAME Conv2D with
 * bias per kernel size, strides `stride`, the kernel sizes sorted, dim / 2, dim / 4, ... channels and the rest for the largest,
 * concatenated in sorted order) and a Transformer of `depth` layers x = short(x) + x, x = mlp(x) + x, x = long(x) + x,
 * x = mlp(x) + x (:196-203).  Attention (:104-180): the module's LayerNorm (eps 1e-5), heads = dim / 32 of width 32, a bias-free
 * 1x1 q|k|v, scores q k^T * 32^-0.5 plus a DynamicPositionBias scalar per in-window offset shared by the heads, softmax, a 1x1
 * to_out with bias; short attention within the local_wsz x local_wsz blocks of the map, long attention within the global_wsz x
 * global_wsz dilated windows (pixels (l1 H / wsz + y, l2 W / wsz + x)).  MLP (:89-102): LayerNorm, 1x1 to 4 dim, exact GELU, 1x1
 * back.  Head: the mean over the map, Dense(num_classes).  Any image whose every stage map (ceil(prev / stride)) is divisible by
 * that stage's local_wsz and global_wsz runs.  The engine runs the cross-scale embedding as one convolution of the largest kernel
 * with the smaller ones nested at its centre, exact for every image size when the stage's kernels share one parity and are all
 * at least its stride; other stages are refused. */
#define VB_CROSSFORMER_STAGES 4
#define VB_CROSSFORMER_MAX_KERNELS 4
typedef struct vb_crossformer_config {
  int32_t struct_size;            /* sizeof(vb_crossformer_config) */
  int32_t dim[VB_CROSSFORMER_STAGES], depth[VB_CROSSFORMER_STAGES], global_wsz[VB_CROSSFORMER_STAGES];
  int32_t local_wsz[VB_CROSSFORMER_STAGES], stride[VB_CROSSFORMER_STAGES];
  int32_t n_kernels[VB_CROSSFORMER_STAGES];                               /* 1 .. VB_CROSSFORMER_MAX_KERNELS */
  int32_t kernels[VB_CROSSFORMER_STAGES][VB_CROSSFORMER_MAX_KERNELS];     /* the first n_kernels[s] entries, any order */
} vb_crossformer_config;

/* CrossFormer.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_CROSSFORMER and
 * its other fields are ignored.  Weights (SURVEY.md App. B) are named by the reference's attribute paths, for stage s, layer l,
 * attention sub-block a in {0 (short), 2 (long)} and MLP sub-block m in {1, 3}:
 *   crossformer_layers.{s}.0.convs.{i}.kernel [k_i, k_i, cin, dim_i] / .bias [dim_i]      (i-th kernel size in sorted order)
 *   crossformer_layers.{s}.1.layers.{l}.{a}.norm.g / .b [1, 1, 1, dim]
 *   ....{a}.to_qkv.kernel [1, 1, dim, 3 * 32 * heads], ....{a}.to_out.kernel [1, 1, 32 * heads, dim] / .bias [dim]
 *   ....{a}.dpb.dpb_layers.{0,3,6}.kernel [2 | dim/4, dim/4] / .bias [dim/4], ....{a}.dpb.dpb_layers.9.kernel [dim/4, 1] / .bias [1],
 *   ....{a}.dpb.dpb_layers.{1,4,7}.gamma / .beta [dim/4]                                  (Keras LayerNormalization, eps 1e-3)
 *   ....{m}.net.0.g / .b [1, 1, 1, dim], ....{m}.net.1.kernel [1, 1, dim, 4 dim] / .bias, ....{m}.net.4.kernel [1, 1, 4 dim, dim] / .bias
 *   to_logits.1.kernel [dim, num_classes] / .bias
 * vb_finalize evaluates every DynamicPositionBias on the host: it depends on the weights alone. */
VB_API int vb_create_crossformer(const vb_config* base, const vb_crossformer_config* cf, int device, vb_handle** out);

/* NesT (nest.py:150-216), appended within ABI 7.  Patch embedding 'b (h p1) (w p2) c -> b h w (p1 p2 c)' and a 1x1 Conv2D(dim)
 * with bias.  `levels` = len(zip(hierarchies, ..., block_repeats)) (nest.py:187): the cast_tuple'd block_repeats truncated to
 * num_hierarchies, or fewer levels when the tuple is shorter; block_repeats[i] is level i's depth.  Level i (bottom first) has
 * width dim * 2^i, heads * 2^i heads of dim_head = dim / heads (inner = dim_head * heads * 2^i may be below the width), and
 * runs on blocks of 2^(levels - 1 - i) x 2^(levels - 1 - i) per map (:208-209): x += pos_emb[:h w] (one scalar per in-block
 * position r * w + c of an h x w block, added to every channel), then block_repeats[i] x [x = Attention(LN(x)) + x,
 * x = MLP(LN(x)) + x] within each block, then Aggregate (Conv2D(3, SAME) with bias to width dim * 2^(i+1), LayerNorm,
 * MaxPool2D(3, 2, SAME)) unless i == num_hierarchies - 1.  Attention (:77-109): a bias-free 1x1 to_qkv, softmax(q k^T *
 * dim_head^-0.5) v per head, a 1x1 to_out with bias.  MLP (:61-75): 1x1 to width * mlp_mult, exact GELU, 1x1 back.  Every
 * LayerNorm is the module's own (eps 1e-5, biased variance, :28-41).  Head: LayerNorm(dim * 2^(num_hierarchies - 1)) per pixel,
 * the mean over the map, Dense(num_classes).  Any image runs whose sides are multiples of patch_size and whose maps are whole
 * blocks of at most seq_len tokens at every level. */
#define VB_NEST_MAX_LEVELS 8
typedef struct vb_nest_config {
  int32_t struct_size;            /* sizeof(vb_nest_config) */
  int32_t patch_size, dim, heads;
  int32_t num_hierarchies;        /* 1 .. VB_NEST_MAX_LEVELS */
  int32_t levels;                 /* 0 .. num_hierarchies: the levels the zip leaves */
  int32_t block_repeats[VB_NEST_MAX_LEVELS];   /* the first `levels` entries */
  int32_t mlp_mult;
  int32_t seq_len;                /* (image_size / patch_size / 2^(num_hierarchies - 1))^2: the length of every pos_emb */
} vb_nest_config;

/* NesT.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_NEST and its other
 * fields are ignored.  Weights (SURVEY.md App. B) are named by the reference's attribute paths, for level i, layer l, width d
 * (d_next the next level's), inner = (dim / heads) * heads * 2^i:
 *   patch_embedding.1.kernel [1, 1, p^2 * channels, dim] / .bias [dim]            (rows in (p1, p2, c) order, c fastest)
 *   nest_layers.{i}.0.pos_emb [seq_len]
 *   nest_layers.{i}.0.layers.{l}.0.norm.g / .b [1, 1, 1, d]
 *   nest_layers.{i}.0.layers.{l}.0.fn.to_qkv.kernel [1, 1, d, 3 * inner]
 *   nest_layers.{i}.0.layers.{l}.0.fn.to_out.0.kernel [1, 1, inner, d] / .bias [d]
 *   nest_layers.{i}.0.layers.{l}.1.norm.g / .b [1, 1, 1, d]
 *   nest_layers.{i}.0.layers.{l}.1.fn.net.0.kernel [1, 1, d, d * mlp_mult] / .bias, ....1.fn.net.3.kernel [1, 1, d * mlp_mult, d] / .bias
 *   nest_layers.{i}.1.ag_layers.0.kernel [3, 3, d, d_next] / .bias [d_next]     (levels with an Aggregate only)
 *   nest_layers.{i}.1.ag_layers.1.g / .b [1, 1, 1, d_next]                      (levels with an Aggregate only)
 *   mlp_head.0.g / .b [1, 1, 1, last_dim], mlp_head.2.kernel [last_dim, num_classes] / .bias
 * A configuration whose last map does not have last_dim = dim * 2^(num_hierarchies - 1) channels (a block_repeats tuple more than
 * one level short) is accepted, as the reference accepts it, and vb_forward refuses it. */
VB_API int vb_create_nest(const vb_config* base, const vb_nest_config* nest, int device, vb_handle** out);

/* RegionViT (regionvit.py:184-263), appended within ABI 7.  dims / depth are the cast_tuple'd 4-tuples (:197-200).  Local tokens:
 * Conv2D(dims[0], 8, stride 4, SAME) of the image, or with tokenize_local_3_conv Conv3x3 s2 -> LayerNormalization -> GELU ->
 * Conv3x3 s2 -> LayerNormalization -> GELU -> Conv3x3 s1 (:210-221).  Regional tokens: 'b (h p1) (w p2) c -> b h w (c p1 p2)',
 * p = local_patch_size * window_size, then a 1x1 Conv2D (:223-226).  Stage s >= 1 applies ONE Downsample Conv2D(dims[s], 3,
 * stride 2, SAME) to both maps (shared weights) and, with use_peg, a depthwise 3x3 PEG plus residual to the local map (:231-240,
 * :257-260).  Then depth[s] R2L layers (:135-182; 4 heads of 32): r = Attention(r) + r over the image's regional tokens; then per
 * lh/rh x lw/rw window [r; window] = Attention([r; window], bias) + [r; window], then MLP + residual, one Attention module used
 * for both.  Attention (:79-116): LayerNormalization, bias-free to_qkv, softmax(q k^T / sqrt(32) + bias) v, to_out with bias;
 * the bias is the window's relative-position Embedding((2 window_size - 1)^2, 4) row (dr + ws - 1) + (dc + ws - 1) (2 ws - 1),
 * zero on the regional token's row and column.  MLP (:64-77): LayerNormalization, Dense(mlp_mult d), exact GELU, Dense(d).  Head
 * (:243-247): the mean over the regional tokens, LayerNormalization, Dense(num_classes).  Every LayerNormalization is Keras's
 * (eps 1e-3).  Any image runs whose sides are multiples of p and whose local map at every stage is a whole number of windows of
 * at most window_size x window_size tokens per regional token. */
#define VB_REGIONVIT_STAGES 4
typedef struct vb_regionvit_config {
  int32_t struct_size;            /* sizeof(vb_regionvit_config) */
  int32_t dims[VB_REGIONVIT_STAGES], depth[VB_REGIONVIT_STAGES];
  int32_t window_size, local_patch_size;
  int32_t tokenize_local_3_conv, use_peg;   /* 0 / 1 */
  int32_t mlp_mult;               /* 4 (regionvit.py:65) */
} vb_regionvit_config;

/* RegionViT.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_REGIONVIT and its
 * other fields are ignored.  Weights (SURVEY.md App. B), for stage s, layer l, width d = dims[s], p = local_patch_size *
 * window_size, t = (2 window_size - 1)^2:
 *   local_encoder.kernel [8, 8, channels, dims[0]] / .bias, or with tokenize_local_3_conv local_encoder.{0,3,6}.kernel [3, 3,
 *     channels | dims[0], dims[0]] / .bias and local_encoder.{1,4}.gamma / .beta [dims[0]]
 *   region_encoder.1.kernel [1, 1, channels * p^2, dims[0]] / .bias   (rows in (c, p1, p2) order, c slowest)
 *   region_layers.{s}.0.conv.kernel [3, 3, dims[s - 1], d] / .bias [d]               (s >= 1)
 *   region_layers.{s}.1.proj.kernel [3, 3, 1, d] / .bias [d]                         (s >= 1 with use_peg)
 *   region_layers.{s}.2.local_rel_pos_bias.embeddings [t, 4]
 *   region_layers.{s}.2.layers.{l}.0.norm.gamma / .beta [d], ....0.to_qkv.kernel [d, 384], ....0.to_out.kernel [128, d] / .bias
 *   region_layers.{s}.2.layers.{l}.1.net.0.gamma / .beta [d], ....1.net.1.kernel [d, mlp_mult d] / .bias, ....1.net.4.kernel
 *     [mlp_mult d, d] / .bias
 *   to_logits.1.gamma / .beta [dims[3]], to_logits.2.kernel [dims[3], num_classes] / .bias
 * vb_finalize stores each stage's Embedding transposed to [4][(2 ws - 1)^2] with the row offset slowest, the index convention of
 * the windowed attention kernels. */
VB_API int vb_create_regionvit(const vb_config* base, const vb_regionvit_config* rv, int device, vb_handle** out);

/* ATS-ViT (ats_vit.py:260-318, adaptive token sampling), appended within ABI 7.  Layer L samples at most
 * max_tokens_per_depth[L] tokens when the batch's padded token count exceeds it (ats_vit.py:213); the first `depth` entries are
 * used, non-increasing and positive (the reference's assert messages). */
#define VB_ATS_MAX_DEPTH 64
typedef struct vb_ats_vit_config {
  int32_t struct_size;            /* sizeof(vb_ats_vit_config) */
  int32_t max_tokens_per_depth[VB_ATS_MAX_DEPTH];
} vb_ats_vit_config;

/* ats_vit.ViT.__init__: `base` supplies the ViT fields (precision, image / patch sizes, channels, num_classes, dim, depth, heads,
 * dim_head, mlp_dim, max_batch); its kind must be VB_KIND_ATS_VIT, the pool is always the cls row.  Weights are ViT's names and
 * shapes (SURVEY.md App. B), to_out always present.  Images may have at most 65,535 patches.  The sampling noise is
 * u = (word 0 of Philox4x32-10 >> 8) * 2^-24 with the 64-bit seed as key and the counter (j | k << 16, b, d_lo, d_hi): j the
 * column of the reference's left-padded [b, K, n - 1] noise tensor, k the draw, b the image, d a 64-bit counter on the device
 * that advances once per layer that samples.  The seed is 0 at creation. */
VB_API int vb_create_ats_vit(const vb_config* base, const vb_ats_vit_config* ats, int device, vb_handle** out);
/* Sets the Philox key and resets the draw counter d to 0 (waits for the device first). */
VB_API int vb_ats_set_seed(vb_handle* h, uint64_t seed);
/* vb_forward (same graph capture and replay) plus the returned token ids: logits [batch, num_classes], token_ids
 * int32 [batch, P - 1] and count (one int32) in host memory, P - 1 the most tokens the last layer can keep.  Columns [0, count) are
 * the reference's `token_ids[:, 1:] - 1` (ats_vit.py:315): each image's kept patch ids in ascending order, left-padded with -1;
 * the columns from count on are -1.  Results depend on the whole batch (through the padded length), as in the reference. */
VB_API int vb_forward_ats(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* logits,
                          int32_t* token_ids, int32_t* count, void* stream);
/* After a forward: whether layer `layer` sampled (*sampled = 1 when the batch's token count exceeded K there), the positions its K
 * draws chose, draws int32 [batch, K] (argmax + 1 in the reference's left-padded layout; all -1 when it did not sample), and the
 * tokens each image kept after it, counts int32 [batch].  A layer whose input can never exceed K is refused. */
VB_API int vb_ats_last_draws(vb_handle* h, int32_t layer, int32_t* draws, int32_t* counts, int32_t* sampled);
/* One ATS sampling step on its own (the engine's ats_sample): qkv float32 [B * P, ld] fused q|k|v rows of B images at pitch P
 * (head h at columns h*dh, HD + h*dh, 2 HD + h*dh), rows int32 [B] the live rows of each image (cls + its c_b tokens; C = the
 * maximum c_b), K draws per image with the Philox key `seed` and draw counter `counter`, scale the softmax scale.  Outputs:
 * sel int32 [B, 1 + min(P - 1, K)] (0, then the kept compact indices in ascending order), rows_new int32 [B] and draws int32
 * [B, K] (argmax + 1 in the left-padded layout; -1 when C <= K and nothing was drawn).  bf16 rounds qkv to bfloat16 first. */
VB_API int vb_op_ats_sample(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t P, int32_t heads, int32_t dh, float scale,
                            const int32_t* rows, int32_t K, uint64_t seed, uint64_t counter, int32_t* sel, int32_t* rows_new,
                            int32_t* draws);
/* Plain attention over fused q|k|v rows (qkv float32 [B * n, ld]) with image b's keys j >= nk_img[b] masked (weight 0), scale
 * dh^-0.5: the dim_head-64 flash kernels in bf16 (resident for n <= 256, streaming above), else the materialised-scores path.
 * out float32 [B * n, ldo]; every row is written, the rows of masked queries too (finite). */
VB_API int vb_op_masked_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t n, int32_t heads, int32_t dh,
                                  const int32_t* nk_img, float* out, int32_t ldo, int32_t iters, float* elapsed_ms);

/* The small-dataset ViT (vit_for_small_dataset.py:159-215: shifted patch tokens and locality self-attention), appended within
 * ABI 7.  vb_create with kind VB_KIND_SMALL_DATASET_VIT: the ViT fields of vb_config are the whole configuration (patch_h ==
 * patch_w, channels 3, pool cls or mean).  Weights are ViT's names and shapes (SURVEY.md App. B), to_out always present, plus
 * patch_norm.gamma / .beta [p^2 * 15] and patch.kernel [p^2 * 15, dim] / .bias (SPT's LayerNormalization and Dense over the
 * (p1, p2, view, c) vector of the image and its four one-pixel shifts) and layers.L.temperature, a scalar (shape (), ndim 0):
 * layer L's softmax scale is exp(temperature) and each token's own key is masked.  vb_forward only: the stage entries and
 * vb_forward_distill refuse the handle. */
/* SPT on its own, plus the cls row and positions (the engine's embedding): img float32 NHWC [B, H, W, 3], patch size p; gamma /
 * beta [p^2 * 15], kernel [p^2 * 15, dim], bias [dim]; cls [dim] and pos [(1 + np) * dim] (either may be NULL: zero).  out float32
 * [B, 1 + np, dim]: row 0 = cls + pos[0], row 1 + t = Dense(LayerNorm(patch t)) + pos[1 + t].  bf16 runs the LayerNorm folded
 * into the wgmma GEMM over rows zero-padded to a multiple of 64 columns, fp32 the LayerNorm kernel and the fp32 GEMM. */
VB_API int vb_op_spt(int32_t precision, const float* img, int32_t B, int32_t H, int32_t W, int32_t p, int32_t dim, const float* gamma,
                     const float* beta, const float* kernel, const float* bias, const float* cls, const float* pos, float* out);
/* Locality self-attention over fused q|k|v rows (qkv float32 [B * n, ld], head h at columns h*dh, HD + h*dh, 2 HD + h*dh): scores
 * q.k * scale with each query's own key masked (weight 0), softmax, times v.  n >= 2.  bf16: the dim_head-64 flash kernels
 * (resident for n <= 256, streaming above), heads narrower than 64 (dh % 8 == 0) zero-padded to 64 as the engine's layers are;
 * other widths and fp32: the materialised-scores path.  out float32 [B * n, ldo]. */
VB_API int vb_op_lsa_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t n, int32_t heads, int32_t dh,
                               float scale, float* out, int32_t ldo, int32_t iters, float* elapsed_ms);

/* Replaces Keras variable assignment: one call per weight, names/shapes/layouts per SURVEY.md App. B
 * (Dense kernel [in,out], float32).  shape/ndim are checked against the config. */
VB_API int vb_set_weight(vb_handle* h, const char* name, const float* host_data, const int64_t* shape, int32_t ndim);

/* Number of weights the config expects, and the name/shape of the i-th (for the host side to enumerate). */
VB_API int vb_num_weights(vb_handle* h);
VB_API int vb_weight_info(vb_handle* h, int32_t index, const char** name, int64_t* shape4, int32_t* ndim);

/* Packs weights for the device (bf16 K-major copies, folded constants).  Fails if a weight is missing. */
VB_API int vb_finalize(vb_handle* h);

/* Replaces <Model>.call(img) (vit.py:159-177, deepvit.py:139-157, cait.py:180-194, cross_vit.py:290-303)
 * with inference semantics (dropout = identity).  img: NHWC float32 [batch,h,w,channels] in host or device
 * memory (img_mem); logits: float32 [batch,num_classes] written to host or device memory (logits_mem).
 * stream: a cudaStream_t (may be NULL = default stream).  With device buffers the call is asynchronous on
 * `stream`; with a host logits buffer it returns after the copy completes.
 * h, w may be smaller than the configured image (pos_embedding[:, :n+1] truncation, vit.py:165).
 * On a stream other than NULL / cudaStreamLegacy the forward of one (image pointer, logits pointer, batch, h, w, stream)
 * combination runs eagerly on its first call, is captured into a CUDA graph on its second and replayed from the third on
 * (vb_graph_stats counts this).  Every call of a handle uses the same workspace, so calls on different streams must be
 * ordered by the caller (an event or a synchronisation between them). */
VB_API int vb_forward(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
               float* logits, int32_t logits_mem, void* stream);

/* Replaces model.transformer(tokens) (vit.py:99-104) for ViT / DeepViT with an arbitrary token count n,
 * the entry the reference's wrappers use (mae.py:69, simmim.py:116, mpp.py:212).
 * tokens/out: float32 [batch, n, dim]. */
VB_API int vb_forward_tokens(vb_handle* h, const float* tokens, int32_t tokens_mem, int32_t batch, int32_t n,
                      float* out, int32_t out_mem, void* stream);

/* DistillMixin.call with a distillation token (reference: distill.py:16-45; DistillableViT distill.py:47-58 on a ViT handle,
 * DistillableT2TViT distill.py:61-72 on a T2TViT handle): patch embedding (T2T: the soft splits and the Dense) + cls +
 * positions, the token appended as the LAST row, the transformer over n + 2 rows, then
 * logits = mlp_head(pool(x[:, :-1])) and distill_out = x[:, -1].  A T2TViT handle created with depth 0 (for an injected
 * transformer) holds no transformer and is refused.
 * distill_token: HOST float32 [dim] (the caller's trainable variable, distill.py:133).  logits [batch, num_classes] and
 * distill_out [batch, dim] live in `out_mem` memory.  img as in vb_forward.
 * LeViT with a distillation head (levit.py:210,220-224): distill_token must be NULL; logits [batch, num_classes] =
 * mlp_head(pool(x)) and distill_out [batch, num_distill_classes] = distill_head(pool(x)). */
VB_API int vb_forward_distill(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                       const float* distill_token, float* logits, float* distill_out, int32_t out_mem, void* stream);

/* ---- the stages of <Model>.call on their own (SURVEY.md 8f f1/f4): the attribute surface the reference's wrappers and the
 * injected-transformer shell use.  ViT / DeepViT / parallel ViT / CaiT / patch-merger ViT / T2TViT; not CrossViT, CCT, LeViT,
 * CvT, Twins-SVT, CrossFormer, NesT or RegionViT. */

/* Number of token rows vb_forward_embed produces for an img_h x img_w image (patches + cls where the model has one);
 * negative on error. */
VB_API int vb_embed_rows(vb_handle* h, int32_t img_h, int32_t img_w);

/* Everything `call` does before `self.transformer` (vit.py:160-166, cait.py:181-184, t2t.py:97-103, efficient.py:40-45,
 * vit_with_patch_merger.py:175-179): patch embedding (T2T: the whole tokens-to-token module), cls token, positions.
 * tokens: float32 [batch, vb_embed_rows, dim]. */
VB_API int vb_forward_embed(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                     float* tokens, int32_t tokens_mem, void* stream);

/* Everything `call` does after `self.transformer` (vit.py:170-175, efficient.py:48-55): pooling (cls row / mean over
 * the n rows, per the config) + mlp_head (LayerNorm, Dense).  tokens float32 [batch, n, dim] -> logits [batch, num_classes].
 * With n == 1 this is `model.mlp_head(x)`. */
VB_API int vb_forward_head(vb_handle* h, const float* tokens, int32_t tokens_mem, int32_t batch, int32_t n, float* logits,
                    int32_t logits_mem, void* stream);

/* `patch_embedding.layers[0]` (the einops Rearrange, vit.py:142; mae.py:37 `to_patch`): img -> float32
 * [batch, num_patches, patch_h*patch_w*channels].  Not for T2TViT. */
VB_API int vb_to_patch(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                float* patches, int32_t patches_mem, void* stream);

/* `patch_embedding.layers[1]` / `.layers[-1]` (the Dense, vit.py:143; mae.py:37 `patch_to_emb`, mpp.py:200):
 * patches float32 [rows, patch_dim] -> float32 [rows, dim] (patch_dim = the Dense's input width; T2T: the last soft split's). */
VB_API int vb_patch_to_emb(vb_handle* h, const float* patches, int32_t patches_mem, int32_t rows, float* out, int32_t out_mem,
                    void* stream);

/* ---- data parallel (SURVEY.md 8e): one handle per GPU (one process or thread each), the batch sharded contiguously, the
 * forward free of communication, ONE in-place NCCL all-gather of the fp32 logits at the end.  The reference has no
 * distributed path; these entries are what its maintainer would call from a multi-process launcher.  NCCL is loaded at
 * vb_dp_init time with dlopen ($VB_NCCL_LIB, else libnccl.so.2): the library itself has no load-time NCCL dependency. ------ */

/* Rank 0: fill id128 (128 bytes, an ncclUniqueId) and hand it to every rank by any transport (file, socket, MPI, gloo). */
VB_API int vb_dp_unique_id(void* id128);

/* Every rank (collective; blocks until all `world` ranks arrive): joins the handle's device to the communicator. */
VB_API int vb_dp_init(vb_handle* h, const void* id128, int32_t rank, int32_t world);

/* vb_forward on this rank's shard of `local_batch` images, its logits written straight into rows
 * [rank*local_batch, (rank+1)*local_batch) of `gathered` (DEVICE float32 [world*local_batch, num_classes]), then
 * ncclAllGather in place on `stream`.  Asynchronous on `stream`. */
VB_API int vb_forward_allgather(vb_handle* h, const float* img, int32_t img_mem, int32_t local_batch, int32_t img_h, int32_t img_w,
                         float* gathered, void* stream);

/* Kernels launched by this handle's most recent forward call. */
VB_API int64_t vb_last_launch_count(vb_handle* h);

/* CUDA-graph activity of vb_forward on this handle, cumulative since vb_create: forwards captured into a graph (the second call
 * of a key on a capturable stream), forwards served by replaying one, and captures that failed -- that key then runs eagerly
 * until its graph is dropped.  *last_failure: the reason of the most recent failed capture ("" if none); valid until the
 * handle's next vb_forward or vb_destroy.  Any pointer may be NULL. */
VB_API int vb_graph_stats(vb_handle* h, int64_t* captures, int64_t* replays, int64_t* failures, const char** last_failure);

/* Which attention kernels served the most recent attention call made on the calling thread since the previous
 * vb_last_attention_path call (which it resets): VB_ATTN_PATH_NONE if there was none.  FLASH: attn_flash_kernel; CLS:
 * attn_cls_kernel (one query row); ROWS: scores_stripe / mid_rows / pv_rows (head mixing, 8 or 16 heads, <= 256 keys);
 * MID_FUSED: scores_mma / mid_fused / pv_mma (bf16 tensor-core scores, every head's scores in shared memory); SIMT:
 * attn_scores / attn_softmax / attn_pv (+ attn_head_mix), every fp32 call and the bf16 fallback. */
#define VB_ATTN_PATH_NONE 0
#define VB_ATTN_PATH_FLASH 1
#define VB_ATTN_PATH_CLS 2
#define VB_ATTN_PATH_ROWS 3
#define VB_ATTN_PATH_MID_FUSED 4
#define VB_ATTN_PATH_SIMT 5
VB_API int32_t vb_last_attention_path(void);

/* Per-kernel-class device timing (CUDA events recorded on the launch stream around every launch of the class)
 * for the roofline report.  Classes: 0 wgmma GEMM (plain / LayerNorm-folded epilogue: to_qkv, to_q, to_kv), 1 attention,
 * 2 LayerNorm / row statistics, 3 im2col, 4 other (SIMT fallbacks), 5 wgmma GEMM with GELU epilogue (fc1),
 * 6 wgmma GEMM with residual epilogue (patch embed, to_out, fc2).
 * LeViT: the stem's unfold is 3 and its convolutions 0; the q / k|v projections and the shrink blocks' to_out are 0, the biased
 * attention 1, the hard-swish fc1 5, the residual to_out / fc2 6; the even-pixel gather is 4 and the average pool 2.
 * CvT: the stems' unfold is 3 and their convolutions 0, the stem LayerNorm (and its row statistics) and the average pool 2; the
 * depthwise q / k|v convolutions (one launch per block) are 4, the pointwise projections 0, attention 1, the LayerNorm-folded GELU
 * fc1 5, the residual to_out / fc2 6 (the fp32 engine adds its separate PreNorm LayerNorms to 2).
 * Twins-SVT: the patch embeddings' unfold and the global to_kv's patch rows are 3; the patch-embedding convolutions, the fused
 * local q|k|v, the global to_q and to_kv are 0; local and global attention 1 (a windowed attention off the flash kernel adds its
 * row permutations to 4); the PEG depthwise convolution (one per stage) 4; the LayerNorm-folded GELU fc1 5; the residual to_out /
 * fc2 6; row statistics and the average pool 2 (the fp32 engine adds its separate LayerNorms to 2).
 * CrossFormer: the cross-scale embeddings' unfold is 3 and their convolution 0; the LayerNorm-folded q|k|v (or v alone for
 * one-token windows) 0; short and long attention 1 (off the flash kernel the row permutations are 4); the LayerNorm-folded GELU
 * fc1 5; the residual to_out / fc2 6; the average pool 2 (the fp32 engine adds its separate LayerNorms to 2).
 * NesT: the patch embedding's and the aggregations' unfold is 3 and their convolutions 0; the LayerNorm-folded q|k|v 0; block
 * attention 1 (off the flash kernel the row permutations are 4); the LayerNorm-folded GELU fc1 5; the residual to_out / fc2 6;
 * the level-0 position add and the aggregation tails (LayerNorm, max-pool, position add) 4; the head's LayerNorm and mean 2 (the
 * fp32 engine adds its separate LayerNorms to 2).
 * RegionViT: the encoders' and the Downsample's unfold is 3 and their convolutions 0; the LayerNorm-folded q|k|v 0; the regional attention and the R2L attention 1 (off the flash kernel
 * the row gathers are 4); the LayerNorm-folded GELU fc1 5; the residual to_out / fc2 6; row statistics, the head's LayerNorm
 * and mean 2; the PEG 4 (the fp32 engine adds its separate LayerNorms to 2).
 * MAE / SimMIM: the kept-patch gather (patch vectors and position rows) is 3; the patch GEMM 6; the encoder's and decoder's layers
 * as ViT's (0, 1, 5, 6, 2); enc_to_dec and to_pixels 0 (off the wgmma path 4); the mask kernel, the decoder-input assembly, SimMIM's
 * mask-token rows, the row gathers, the pred / masked_patches outputs and the loss reductions 4.
 * MPP: the corrupted-patch gather is 3; the patch GEMM 6; the encoder's layers as ViT's; to_bits 0 (off the wgmma path 4); the mask
 * kernel, the corruption draws, the masked-row gather, the outputs and the loss reduction 4.
 * vb_profile_read synchronises the device and returns accumulated milliseconds, algorithmic FLOPs, algorithmic
 * bytes and launch counts per class (arrays of VB_PROF_NUM); reset != 0 clears the accumulators. */
#define VB_PROF_NUM 7
VB_API int vb_profile_enable(vb_handle* h, int32_t on);
VB_API int vb_profile_read(vb_handle* h, double* ms, double* flops, double* bytes, int64_t* calls, int32_t reset);

VB_API const char* vb_last_error(vb_handle* h);
VB_API void vb_destroy(vb_handle* h);

/* ---- single-operator entry points (used by the parity tests and the per-kernel benchmarks) -------------
 * All buffers are HOST float32; bf16 variants round operands to bf16 (RNE) on the way in.
 * *elapsed_ms (may be NULL) receives the average device time per launch over `iters` launches (CUDA events). */

/* out[M,N] = epi(a[M,K] x w[K,N]): epi = (+bias[N]) -> exact-erf GELU (gelu!=0) -> (*scale[N]) -> (+res[M,N]).
 * Any of bias/scale/res may be NULL.  precision BF16 runs the wgmma kernel, FP32 the SIMT kernel. */
VB_API int vb_op_linear(int32_t precision, const float* a, const float* w, const float* bias, const float* scale,
                 const float* res, int32_t gelu, float* out, int32_t M, int32_t N, int32_t K, int32_t iters,
                 float* elapsed_ms);

/* Multi-head attention core (vit.py:77-82): q [B,nq,h*dh], k,v [B,nk,h*dh] -> out [B,nq,h*dh];
 * variant 0 = plain, 1 = DeepViT re-attention (mix [h,h] + LayerNorm over heads, gamma/beta [h]; deepvit.py:83-84),
 * 2 = CaiT talking heads (mix_pre, mix_post [h,h]; cait.py:123-125). */
VB_API int vb_op_attention(int32_t precision, int32_t variant, const float* q, const float* k, const float* v,
                    const float* mix_a, const float* mix_b, const float* ln_gamma, const float* ln_beta,
                    float* out, int32_t B, int32_t nq, int32_t nk, int32_t heads, int32_t dim_head, int32_t iters,
                    float* elapsed_ms);

/* LayerNorm over the last axis, eps 1e-3 (vit.py:18): x [M,D] -> out [M,D]. */
VB_API int vb_op_layernorm(int32_t precision, const float* x, const float* gamma, const float* beta, float* out,
                    int32_t M, int32_t D, int32_t iters, float* elapsed_ms);

/* PatchMerger.call (vit_with_patch_merger.py:49-55): x [B,n,D] -> LayerNorm -> softmax(queries [nt,D] . x^T * D^-0.5) . x
 * -> out [B,nt,D]. */
VB_API int vb_op_patch_merger(int32_t precision, const float* x, const float* gamma, const float* beta, const float* queries,
                       float* out, int32_t B, int32_t n, int32_t D, int32_t nt, int32_t iters, float* elapsed_ms);

/* PreNorm + Dense as the bf16 engine runs it (vit.py:18-22 followed by vit.py:39 / :59): LayerNorm over the last axis
 * (eps 1e-3) FOLDED into the following Dense -- gamma scaled into the packed weights, the per-row (mean, rstd) reduced in
 * the GEMM epilogue from (sum, sumsq) partials of the bf16 rows.  x [M,K], w [K,N] (Keras layout), bias [N] or NULL,
 * out [M,N] = act(LN(x) w + bias), act = exact-erf GELU when gelu != 0.  bf16 engine only; N % 64 == 0, K % 64 == 0. */
VB_API int vb_op_ln_linear(const float* x, const float* gamma, const float* beta, const float* w, const float* bias,
                    int32_t gelu, float* out, int32_t M, int32_t N, int32_t K, int32_t iters, float* elapsed_ms);

/* ---- the kernels in the operand layouts the engine itself uses (strided rows, in-place residuals, row statistics,
 * fused q|k|v rows, head-padded attention).  Same conventions as above; a result is that of the FIRST launch (later timed
 * launches may update an in-place residual again). ------------------------------------------------------------------------ */

/* bf16 wgmma GEMM: out[m, out_off + n] = epi(sum_k a[m, k] wt[n, k]), m < M, n < N, k < K.
 *   a       [M, lda], lda >= K: only columns < K are read.
 *   wt      the weight in its K-major packed form [b_rows, ldw] (b_rows = 0: N); rows [b_rows, N) read as zero.
 *   out     [M, ldc]: the whole buffer is uploaded (rounded to bf16 unless out_f32) and downloaded again, so columns the
 *           GEMM does not write come back unchanged.  out_f32 != 0: fp32 output, plain or bias epilogue only.
 *   epi     (+bias[N]) -> activation -> (*scale[N]) -> (+res[m, n]); gelu: 0 none, 3 SiLU (with a bias or the folded
 *           LayerNorm), any other value exact-erf GELU (as every nonzero value meant before SiLU).  res == out: the residual is the
 *           output region itself (in place, ldr must equal ldc); otherwise res is a separate [M, ldr] buffer at column 0.
 *   ln_stats, ln_c1: folded LayerNorm of the A rows (as vb_op_ln_linear runs it): wt must hold gamma-scaled weights, bias the
 *           c2 = beta.W + bias term, ln_c1[N] the row sums of wt, ln_stats [K/64][M] (sum, sumsq) float pairs of the rows.
 *   stats_out (may be NULL): receives [N/64][M] (sum, sumsq) float pairs of each 64-column chunk of the stored bf16 rows.
 * Every leading dimension and out_off must be a multiple of 8; N % 64 == 0, K % 8 == 0. */
VB_API int vb_op_gemm(const float* a, int32_t lda, const float* wt, int32_t ldw, int32_t b_rows, const float* bias,
                      const float* scale, int32_t gelu, const float* res, int32_t ldr, const float* ln_stats, const float* ln_c1,
                      float* out, int32_t ldc, int32_t out_off, int32_t out_f32, float* stats_out, int32_t M, int32_t N, int32_t K,
                      int32_t iters, float* elapsed_ms);

/* Multi-head attention with explicit layouts, run exactly as the engine dispatches it (fused kernels first, the
 * materialised-scores path otherwise).  q: [B*nq, ldq], head h of row i at columns [h*dh, (h+1)*dh).  kv == NULL: k and v
 * are the columns [k_off, ..) and [v_off, ..) of the q buffer (the fused [q|k|v] rows, nk == nq, pitch ldq); otherwise of
 * kv [B*nk, ldkv] (the [k|v] rows of class / cross attention).  out: [B*nq, ldo], uploaded and downloaded whole.
 * dh: the activation head width; scale: softmax scale, <= 0 means dh^-0.5 (a head-padded layer passes its model
 * dim_head^-0.5).  variant / mixes as vb_op_attention. */
VB_API int vb_op_attention_ex(int32_t precision, int32_t variant, const float* q, int32_t ldq, const float* kv, int32_t ldkv,
                              int32_t k_off, int32_t v_off, const float* mix_a, const float* mix_b, const float* ln_gamma,
                              const float* ln_beta, float* out, int32_t ldo, int32_t B, int32_t nq, int32_t nk, int32_t heads,
                              int32_t dh, float scale, int32_t iters, float* elapsed_ms);

/* LeViT attention (levit.py:119-139) as the engine runs it: softmax(q k^T * scale + bias) v, then GELU (gelu_out != 0).
 * q [B*nq, ldq], k [B*nk, ldk], v [B*nk, ldv] (head h at columns [h*dh, (h+1)*dh)); out [B*nq, ldo], uploaded and downloaded
 * whole.  nk = fmap^2 keys on a fmap x fmap grid; nq = ceil(fmap / q_step)^2 queries on its pixels (q_step*r, q_step*c).
 * pos_bias: the Embedding table [fmap^2, heads] (levit.py:101); the bias of (i, j) is pos_bias[|dr| * fmap + |dc|, h] / scale
 * (:117), packed as vb_finalize packs it.  scale > 0 (the model's dim_key^-0.5).  The flash kernel serves dh == 64 (bf16);
 * other widths and every fp32 call take the materialised-scores path (vb_last_attention_path tells which). */
VB_API int vb_op_attention_bias(int32_t precision, const float* q, int32_t ldq, const float* k, int32_t ldk, const float* v,
                                int32_t ldv, const float* pos_bias, float* out, int32_t ldo, int32_t B, int32_t heads, int32_t dh,
                                int32_t fmap, int32_t q_step, float scale, int32_t gelu_out, int32_t iters, float* elapsed_ms);

/* CvT's depthwise projections (cvt.py:79-92,111-115) as the engine runs them, for one block: y = LN(x) over the C channels (eps
 * 1e-5, ln_gamma / ln_beta [C]), q = BN_q(dw_q(y)) with stride 1 and kv = BN_kv(dw_kv(y)) with stride kv_stride (1 or 2), k x k
 * (k <= 7) TF SAME depthwise convolutions whose padding is zeros of y.  x: [B, H, W, C] NHWC; wq / wkv: the depthwise kernels
 * [k, k, 1, C]; bn_q / bn_kv: the BatchNormalization [4, C] = gamma, beta, moving_mean, moving_variance (folded on the host as
 * vb_finalize does); q [B, H, W, C], kv [B, ceil(H/s), ceil(W/s), C].  bf16 (precision 1): x in bf16 with C zero-padded to a
 * multiple of 64, the LayerNorm applied on load from the rows' (sum, sumsq) statistics; fp32: a separate LayerNorm, then the
 * convolutions.  All buffers are host memory. */
VB_API int vb_op_dwconv(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* ln_gamma,
                        const float* ln_beta, int32_t k, int32_t kv_stride, const float* wq, const float* bn_q, const float* wkv,
                        const float* bn_kv, float* q, float* kv, int32_t iters, float* elapsed_ms);

/* Twins-SVT's local attention (twins_svt.py:135-156) as the engine runs it: the map's p x p windows each attend within themselves.
 * qkv: the fused q|k|v rows of a pixel-major [B, H, W] map, [B*H*W, ld] with q, k and v at columns [0, heads*dh), [heads*dh,
 * 2*heads*dh) and [2*heads*dh, 3*heads*dh), head h at [h*dh, (h+1)*dh) of each; H and W multiples of p; out [B*H*W, ldo]
 * pixel-major, uploaded and downloaded whole.  Scale dh^-0.5.  bf16 with dh == 64 runs the windowed flash kernel on the rows in
 * place; every fp32 call and any shape it refuses permute the rows to window-major order, run the materialised-scores path and
 * permute back (vb_last_attention_path tells which). */
VB_API int vb_op_window_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t p,
                                  int32_t heads, int32_t dh, float* out, int32_t ldo, int32_t iters, float* elapsed_ms);

/* CrossFormer's attention (crossformer.py:141-172) as the engine runs it: vb_op_window_attention's layout with windows of
 * wsz x wsz tokens, contiguous blocks (is_long == 0) or the dilated windows of the long attention (is_long != 0: token (l1, l2) of
 * window (y, x) is the pixel (l1 H / wsz + y, l2 W / wsz + x)), and every score plus table[(dr + wsz - 1) * (2 wsz - 1) + dc + wsz
 * - 1] for the in-window offset (dr, dc) of query and key; table: (2 wsz - 1)^2 floats, shared by the heads.  Scale dh^-0.5.  bf16
 * with dh 32 or 64 and wsz <= 32 runs the windowed-bias flash kernel in place; every fp32 call and any shape it refuses permute
 * the rows, run the materialised-scores path with the table added and permute back (vb_last_attention_path tells which). */
VB_API int vb_op_window_bias_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t wsz,
                                       int32_t is_long, int32_t heads, int32_t dh, const float* table, float* out, int32_t ldo,
                                       int32_t iters, float* elapsed_ms);

/* NesT's block attention (nest.py:93-109) as the engine runs it: vb_op_window_attention's layout with contiguous bh x bw blocks
 * (H a multiple of bh, W of bw; token r * bw + c of a block), each attending within itself.  Scale dh^-0.5.  bf16 with dh 32 or
 * 64 runs the windowed flash kernel in place; every fp32 call and any other dh permute the rows to block-major order, run the
 * materialised-scores path and permute back (vb_last_attention_path tells which). */
VB_API int vb_op_block_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t bh,
                                 int32_t bw, int32_t heads, int32_t dh, float* out, int32_t ldo, int32_t iters, float* elapsed_ms);

/* RegionViT's regional-to-local attention (regionvit.py:143-177) as the engine runs it: qkv [B*lh*lw + B*rh*rw, ld] holds the
 * fused q|k|v rows of the pixel-major local map followed by those of the pixel-major region map (lh = rh * wh, lw = rw * ww,
 * wh and ww <= window_size).  Window (b, wy, wx) attends over its regional row (b * rh + wy) * rw + wx and its wh x ww local
 * rows, scale dh^-0.5, with table[(dr + ws - 1) + (dc + ws - 1) (2 ws - 1), h] (the reference's Embedding layout [(2 ws - 1)^2,
 * heads]) added to the local-local scores.  out [rows, ldo] receives every row's output in place.  bf16 with dh 32 runs the
 * R2L flash kernel; fp32, any other dh and tables past the kernel's shared-memory table gather the windows, run the
 * materialised-scores path and scatter back (vb_last_attention_path tells which). */
VB_API int vb_op_r2l_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t lh, int32_t lw, int32_t rh,
                               int32_t rw, int32_t heads, int32_t dh, const float* table, int32_t window_size, float* out,
                               int32_t ldo, int32_t iters, float* elapsed_ms);

/* NesT's aggregation tail (nest.py:111-123 after the convolution, then :140-142 of the next level) as the engine runs it:
 * x [B, H, W, C] NHWC -> y = LayerNorm(x) over C (eps 1e-5, gamma / beta [C]) -> MaxPool2D(3, 2, 'SAME') -> + pos[(r % bh) * bw
 * + c % bw] on every channel of output pixel (r, c) (pos may be NULL: no add) -> out [B, ceil(H/2), ceil(W/2), C].  bf16
 * (precision 1): x in bf16 with C zero-padded to a multiple of 64, the LayerNorm applied on load from the rows' (sum, sumsq)
 * statistics, and stats_out (may be NULL) receives the output rows' [Cp/64][rows] (sum, sumsq) float pairs; fp32: a separate
 * LayerNorm, then the pool (stats_out unused).  All buffers are host memory. */
VB_API int vb_op_nest_aggregate(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, const float* gamma,
                                const float* beta, const float* pos, int32_t bh, int32_t bw, float* out, float* stats_out,
                                int32_t iters, float* elapsed_ms);

/* MobileViT (mobile_vit.py:209-271), appended within ABI 7.  conv1: Conv_NxN_BN(channels[0], 3, stride 2); stem: MV2 blocks 0-3;
 * trunk: per stage s an MV2 block (4 + s, stride 2) and a MobileViTBlock(dims[s], depths[s], channels[5 + 2 s], kernel_size,
 * (ph, pw), mlp dims[s] * (2, 4, 4)[s]); to_logits: Conv_NxN_BN(last_dim, 1), the mean over pixels, a bias-free Dense.  Conv_NxN_BN
 * is a bias-free SAME Conv2D, BatchNormalization (eps 1e-5, moving statistics) and SiLU.  An MV2 block (:130-170) is [1x1 conv + BN
 * + SiLU when mv2_expand], 3x3 depthwise conv (stride mv2_stride, SAME) + BN + SiLU, 1x1 conv + BN, plus its input when
 * mv2_residual; mv2_in / mv2_hidden / mv2_out are its widths as the host computed them (hidden = int(dim_in * expansion) of the
 * reference's dim_in; mv2_hidden == mv2_in without the expand conv).  A MobileViTBlock (:173-206) runs k x k and 1x1 Conv_NxN_BN to
 * dims[s], then depths[s] pre-norm layers (LayerNormalization eps 1e-3; attention of 4 heads of 8 within each of the ph * pw
 * patch positions, 'b (h ph) (w pw) d -> b (ph pw) (h w) d', scale 8^-0.5, bias-free to_qkv, to_out with bias; MLP Dense, SiLU,
 * Dense), a 1x1 Conv_NxN_BN back to channels[5 + 2 s], the concat with the block's input and a k x k Conv_NxN_BN.  Every trunk map
 * (1/8, 1/16 and 1/32 of the image under SAME's ceil) must be divisible by (ph, pw). */
#define VB_MOBILEVIT_MV2 7
typedef struct vb_mobilevit_config {
  int32_t struct_size;            /* sizeof(vb_mobilevit_config) */
  int32_t channels[10];           /* the reference's channels[0..9] */
  int32_t last_dim;               /* channels[-1] */
  int32_t dims[3], depths[3];
  int32_t kernel_size, ph, pw;
  int32_t mv2_in[VB_MOBILEVIT_MV2], mv2_hidden[VB_MOBILEVIT_MV2], mv2_out[VB_MOBILEVIT_MV2], mv2_stride[VB_MOBILEVIT_MV2];
  int32_t mv2_expand[VB_MOBILEVIT_MV2], mv2_residual[VB_MOBILEVIT_MV2];   /* 0 / 1 */
} vb_mobilevit_config;

/* MobileViT.__init__: `base` supplies precision, channels (3), num_classes and max_batch; its kind must be VB_KIND_MOBILEVIT and
 * its other fields are ignored.  Weights (SURVEY.md App. B) are named by the reference's attribute paths; BN stands for the
 * BatchNormalization leaves .gamma / .beta / .moving_mean / .moving_variance [width]:
 *   conv1.layers.0.kernel [3, 3, 3, channels[0]], conv1.layers.1 BN
 *   MV2 block i (stem.{i}.conv for i < 4, trunk.{i - 4}.0.conv after), with expand: .0.kernel [1, 1, in, hidden], .1 BN,
 *     .3.kernel [3, 3, 1, hidden], .4 BN, .6.kernel [1, 1, hidden, out], .7 BN; without: .0.kernel [3, 3, 1, hidden], .1 BN,
 *     .3.kernel [1, 1, hidden, out], .4 BN
 *   trunk.{s}.1.conv1.layers.0.kernel [k, k, channels[4 + 2 s], c], .1 BN (c = channels[5 + 2 s]); conv2 [1, 1, c, dims[s]];
 *     conv3 [1, 1, dims[s], c]; conv4 [k, k, c + channels[4 + 2 s], c]; each with its .layers.1 BN
 *   trunk.{s}.1.transformer.layers.{l}.0.norm.gamma / .beta, .0.fn.to_qkv.kernel [dims[s], 96], .0.fn.to_out.0.kernel [32,
 *     dims[s]] / .bias, .1.norm.gamma / .beta, .1.fn.net.0.kernel [dims[s], mlp] / .bias, .1.fn.net.3.kernel [mlp, dims[s]] / .bias
 *   to_logits.0.layers.0.kernel [1, 1, channels[9], last_dim], to_logits.0.layers.1 BN, to_logits.2.kernel [last_dim, num_classes]
 * vb_forward only: the stage entries and vb_forward_distill refuse the handle. */
VB_API int vb_create_mobilevit(const vb_config* base, const vb_mobilevit_config* mv, int device, vb_handle** out);
/* MobileViT's MV2 depthwise step as the engine runs it: x [B, H, W, C] NHWC; w the depthwise kernel [3, 3, 1, C]; bn [4, C] =
 * gamma, beta, moving_mean, moving_variance (folded on the host as vb_finalize folds it); out [B, ceil(H/s), ceil(W/s), Cp] =
 * SiLU(BN(dw(x))) with TF SAME padding at stride 1 or 2, Cp = C in fp32 and C rounded up to a multiple of 64 in bf16 (x in bf16
 * at that pitch), columns [C, Cp) as the kernel wrote them.  All buffers are host memory. */
VB_API int vb_op_mv2_dwconv(int32_t precision, const float* x, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride, const float* w,
                            const float* bn, float* out, int32_t iters, float* elapsed_ms);
/* MobileViT's attention (mobile_vit.py:95-107,196-199) as the engine runs it: qkv [B*H*W, ld] the fused q|k|v rows of a
 * pixel-major [B, H, W] map (head h at columns h*dh, HD + h*dh, 2 HD + h*dh, HD = heads * dh); the pixels (y, x) with the same
 * (y % ph, x % pw) attend together, softmax(q k^T * scale) v; out [B*H*W, ldo] pixel-major, uploaded and downloaded whole.  bf16
 * with dh 32 or 64 runs the windowed flash kernel on the rows in place; fp32 and any other shape permute the rows, run the
 * materialised-scores path and permute back (vb_last_attention_path tells which). */
VB_API int vb_op_patch_attention(int32_t precision, const float* qkv, int32_t ld, int32_t B, int32_t H, int32_t W, int32_t ph, int32_t pw,
                                 int32_t heads, int32_t dh, float scale, float* out, int32_t ldo, int32_t iters, float* elapsed_ms);

/* ScalableViT (scalable_vit.py:250-319), appended within ABI 7.  to_patches: Conv2D(dim[0], 7, stride 4, SAME, bias); stage s <
 * num_stages: a Transformer of depth[s] blocks on the dim[s] = dim * 2^s map, its own LayerNorm (eps 1e-5), then (s < num_stages - 1)
 * Downsample: Conv2D(dim[s + 1], 3, stride 2, SAME, bias); the head: the mean over pixels, LayerNormalization (eps 1e-3), Dense.
 * Each block is built [SSA, MLP, PEG (first block only), MLP, IWSA] (:222-231) but unpacked as ssa, ff1, peg, iwsa, ff2 (:236), so
 * it runs x = SSA(LN x) + x, x = MLP(LN x) + x, x = PEG(x), x = MLP(LN x) + x, x = IWSA(LN x) + x, every LN the model's own
 * (biased variance, eps 1e-5).  SSA (:104-143): q a bias-free 1x1 convolution to heads * ssa_dim_key, k and v bias-free r x r
 * stride-r VALID convolutions to heads * ssa_dim_key / ssa_dim_value (r = reduction_factor), softmax(q k^T * ssa_dim_key^-0.5) v,
 * to_out a 1x1 convolution with bias.  IWSA (:145-198): bias-free 1x1 q / k / v, attention within window x window windows (0:
 * the whole map), plus LIM(v), a full 3x3 SAME convolution with bias over v's heads * iwsa_dim_value channels, then to_out.  MLP:
 * 1x1 convolution to ff_expansion_factor * dim[s], exact-erf GELU, 1x1 convolution back, both with bias.  PEG: x + a depthwise 3x3
 * SAME convolution with bias.  Any image size runs whose stage maps (ceil(H / 4), then ceil(/ 2) per stage) are at least
 * reduction_factor on each side and divisible by their window. */
#define VB_SCALABLE_VIT_STAGES 4
typedef struct vb_scalable_vit_config {
  int32_t struct_size;            /* sizeof(vb_scalable_vit_config) */
  int32_t num_stages;             /* 1 to VB_SCALABLE_VIT_STAGES */
  int32_t dim[VB_SCALABLE_VIT_STAGES], depth[VB_SCALABLE_VIT_STAGES], heads[VB_SCALABLE_VIT_STAGES];
  int32_t ssa_dim_key[VB_SCALABLE_VIT_STAGES], ssa_dim_value[VB_SCALABLE_VIT_STAGES], reduction_factor[VB_SCALABLE_VIT_STAGES];
  int32_t iwsa_dim_key[VB_SCALABLE_VIT_STAGES], iwsa_dim_value[VB_SCALABLE_VIT_STAGES];
  int32_t window[VB_SCALABLE_VIT_STAGES];   /* 0: the whole map is one window (window_size None) */
  int32_t ff_expansion_factor;
} vb_scalable_vit_config;

/* ScalableViT.__init__: `base` supplies precision, channels, num_classes and max_batch; its kind must be VB_KIND_SCALABLE_VIT and
 * its other fields are ignored.  Weights (SURVEY.md App. B) are named by the reference's attribute paths (d = dim[s], h = heads[s],
 * the reference's LayerNorm leaves .g / .b of shape [1, 1, 1, d]); block l of stage s is scalable_layers.{s}.0.layers.{l}.{j} with
 * j the construction index:
 *   to_patches.kernel [7, 7, channels, dim[0]] / .bias
 *   j = 0 (SSA): .0.norm.g / .b, .0.fn.to_q.kernel [1, 1, d, h dk], .0.fn.to_k.kernel [r, r, d, h dk], .0.fn.to_v.kernel [r, r, d,
 *     h dv], .0.fn.to_out.0.kernel [1, 1, h dv, d] / .bias
 *   j = 1, 3 (MLP): .norm.g / .b, .fn.net.0.kernel [1, 1, d, f d] / .bias, .fn.net.3.kernel [1, 1, f d, d] / .bias
 *   j = 2 (PEG, l = 0 only): .proj.kernel [3, 3, 1, d] / .bias
 *   j = 4 (IWSA): .4.norm.g / .b, .4.fn.local_interactive_module.kernel [3, 3, h dv, h dv] / .bias, .4.fn.to_q.kernel / .to_k.kernel
 *     [1, 1, d, h dk], .4.fn.to_v.kernel [1, 1, d, h dv], .4.fn.to_out.0.kernel [1, 1, h dv, d] / .bias
 *   scalable_layers.{s}.0.norm.g / .b; scalable_layers.{s}.1.conv.kernel [3, 3, d, 2 d] / .bias (s < num_stages - 1)
 *   mlp_head.1.gamma / .beta [dim[-1]], mlp_head.2.kernel [dim[-1], num_classes] / .bias
 * vb_forward only: the stage entries and vb_forward_distill refuse the handle. */
VB_API int vb_create_scalable_vit(const vb_config* base, const vb_scalable_vit_config* sv, int device, vb_handle** out);

/* PiT (pit.py:158-219) as the reference runs it, appended within ABI 7.  No pooling stage is ever built (`ind < (len(depth) < 1)`
 * is `ind < 0`, pit.py:194), so the model is one token stream of width dim: patch embedding = tf.image.extract_patches(p, stride
 * p / 2, VALID) ((k_row, k_col, c) vectors, c fastest) then Dense(dim); cls row and pos_embedding[:, :n + 1]; the stages in order,
 * stage s a ViT Transformer of depth[s] layers with heads[s] heads of dim_head (pre-norm attention with a bias-free to_qkv, to_out
 * unless heads[s] == 1 and dim_head == dim; pre-norm MLP with exact-erf GELU; Keras LayerNormalization, eps 1e-3); head: the cls
 * row, LayerNormalization, Dense(num_classes).  `stages` counts what the reference's zip(depth, cast_tuple(heads)) leaves. */
#define VB_PIT_MAX_STAGES 8
typedef struct vb_pit_config {
  int32_t struct_size;            /* sizeof(vb_pit_config) */
  int32_t stages;                 /* 0 .. VB_PIT_MAX_STAGES (0: embedding and head only) */
  int32_t depth[VB_PIT_MAX_STAGES], heads[VB_PIT_MAX_STAGES];   /* the first `stages` entries */
} vb_pit_config;

/* PiT.__init__: `base` supplies precision, image_h == image_w (image_size), patch_h == patch_w (patch_size, at least 2: the
 * stride is patch_size / 2), channels, num_classes, dim, dim_head, mlp_dim and max_batch; its kind must be VB_KIND_PIT and its
 * other fields are ignored.  The table has num_patches + 1 rows, num_patches = ((image_size - p) / (p / 2) + 1)^2.  Weights are
 * ViT's names and shapes (SURVEY.md App. B), with layer L counted across the stages in order:
 *   patch.kernel [p^2 * channels, dim] / .bias          patch_embedding.layers[1]
 *   pos_embedding [1, num_patches + 1, dim], cls_token [1, 1, dim]
 *   layers.L.attn_norm.gamma / .beta, layers.L.to_qkv.kernel [dim, 3 heads[s] dim_head]     transformer_layers.{s}.layers.{l}.0
 *     (.norm, .fn.to_qkv)
 *   layers.L.to_out.kernel [heads[s] dim_head, dim] / .bias   ....{l}.0.fn.to_out.layers[0]; absent where heads[s] == 1 and
 *     dim_head == dim
 *   layers.L.ff_norm.gamma / .beta, layers.L.fc1 / .fc2 .kernel / .bias   ....{l}.1 (.norm, .fn.net.layers[0], .fn.net.layers[3])
 *   head_norm.gamma / .beta, head.kernel / .bias        mlp_head.layers[0], mlp_head.layers[1]
 * for stage s and its layer l (L = depth[0] + ... + depth[s - 1] + l).  vb_forward takes any image of at least p x p whose
 * (floor((h - p) / (p / 2)) + 1) (floor((w - p) / (p / 2)) + 1) patches fit the table (the reference reads its first n + 1
 * rows); the stage entries and vb_forward_distill refuse the handle. */
VB_API int vb_create_pit(const vb_config* base, const vb_pit_config* pit, int device, vb_handle** out);

/* Masked image modelling (MAE, mae.py:49-92; SimMIM, simmim.py:82-129), appended within ABI 7: inference semantics, the loss value
 * and what it is computed from.  For an image of n = (h / patch_h) (w / patch_w) patches, num_masked = (int)(masking_ratio * n) in
 * IEEE double (0.29 * 100 gives 28).
 *   Noise: u[b, j] = (word 0 of Philox4x32-10 >> 8) * 2^-24, j < n, with the 64-bit seed as key and the counter (j, b, d_lo, d_hi),
 *   d a 64-bit counter on the device that advances once per forward (graph replays draw fresh masks).  The seed is 0 at creation.
 *   Order: MAE sorts the ids ascending by (u, j) (the reference's argsort); SimMIM descending by u with ties to the smaller j (its
 *   top_k).  The first num_masked ids of that permutation are masked.  With 24-bit noise ties occur (about a quarter of the
 *   calls at n = 196 and batch 256 hold one), so the order is defined exactly.
 *   MAE: tokens = patch_to_emb(kept patches) + pos_embedding[1 + id] (no cls row); the encoder's transformer over the n -
 *   num_masked kept rows; enc_to_dec (a Dense, or the identity when dim == decoder_dim) + decoder_pos_emb[id]; the decoder input is
 *   the num_masked rows mask_token + decoder_pos_emb[masked id] and the kept rows; the decoder (a ViT Transformer of decoder_depth
 *   layers, decoder_heads heads of decoder_dim_head, mlp 4 decoder_dim, no final norm, to_out dropped when decoder_heads == 1 and
 *   decoder_dim_head == decoder_dim); pred = to_pixels(the mask rows).  loss = mean(pred^2): the reference's
 *   tf.reduce_mean(tf.square(pred, masked_patches)) passes masked_patches as tf.square's `name` (mae.py:90).
 *   SimMIM: tokens = patch_to_emb(patches) + pos_embedding[1 + j], the masked rows replaced by mask_token + pos_embedding[1 + j];
 *   the encoder's transformer over all n rows; pred = to_pixels(the encoded rows at the masked ids, in top_k order);
 *   loss = mean(|pred - masked_patches|) / num_masked (simmim.py:128, the extra division is the reference's).
 * VB_MIM_MAX_PATCHES: the most patches per image the mask kernel sorts (in shared memory). */
#define VB_MIM_MAX_PATCHES 4096
typedef struct vb_mim_config {
  int32_t struct_size;            /* sizeof(vb_mim_config) */
  double masking_ratio;           /* in (0, 1) */
  int32_t decoder_dim, decoder_depth, decoder_heads, decoder_dim_head;   /* MAE only */
} vb_mim_config;

/* MAE.__init__ / SimMIM.__init__: `encoder` supplies the encoder ViT's fields (precision, image / patch sizes, channels, dim, depth,
 * heads, dim_head, mlp_dim, max_batch); its kind must be VB_KIND_MAE or VB_KIND_SIMMIM, num_classes and pool are ignored.
 * Weights (SURVEY.md App. B): the encoder's ViT names without cls_token, head_norm.* and head.* -- pos_embedding [1, n_p + 1, dim],
 * patch.kernel [patch_h patch_w channels, dim] / .bias, layers.L.* -- plus
 *   MAE:    mask_token [decoder_dim]; enc_to_dec.kernel [dim, decoder_dim] / .bias (only when dim != decoder_dim);
 *           decoder.layers.L.* (ViT's layer names and shapes at width decoder_dim); decoder_pos_emb.embeddings [n_p + 1, decoder_dim]
 *           (Embedding(num_patches, decoder_dim) with num_patches = pos_embedding.shape[-2]); to_pixels.kernel [decoder_dim,
 *           patch_dim] / .bias
 *   SimMIM: mask_token [dim]; to_pixels.kernel [dim, patch_dim] / .bias
 * with patch_dim = patch_h patch_w channels and n_p the configured patch count. */
VB_API int vb_create_mim(const vb_config* encoder, const vb_mim_config* mim, int device, vb_handle** out);
/* Sets the Philox key of the mask noise and resets the draw counter d to 0 (waits for the device first). */
VB_API int vb_mim_set_seed(vb_handle* h, uint64_t seed);
/* One MAE / SimMIM call: img NHWC float32 [batch, img_h, img_w, channels] in img_mem memory; loss: one float; pred and
 * masked_patches [batch, num_masked, patch_dim] (may be NULL); indices int32 [batch, n], each image's noise permutation with the
 * masked ids first (may be NULL); all outputs in out_mem memory.  Graph capture and replay follow vb_forward's rules, keyed also by
 * which of pred / masked_patches are requested.  Refused: sides not divisible by the patch, more than n_p patches or more than
 * VB_MIM_MAX_PATCHES, and num_masked == 0 (the reference's mean over no rows would be NaN).  An image's masks and pred do not
 * depend on the rest of the batch; the loss is a fixed-order reduction, so eager, captured and replayed calls give the same bits. */
VB_API int vb_forward_mim(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* loss,
                          float* pred, float* masked_patches, int32_t* indices, int32_t out_mem, void* stream);
/* The mask kernel on its own: indices int32 [B, n] (host) for the Philox key `seed` and draw counter `counter`; descending = 0
 * MAE's order, 1 SimMIM's.  1 <= n <= VB_MIM_MAX_PATCHES. */
VB_API int vb_op_mim_mask(int32_t descending, int32_t B, int32_t n, uint64_t seed, uint64_t counter, int32_t* indices);

/* Masked patch prediction (MPP, mpp.py:133-218), appended within ABI 7 on the masked-image-modelling handle: inference semantics
 * and the loss value.  For an image of n = (h / patch) (w / patch) patches:
 *   Mask: k = ceil(mask_prob * n) in IEEE double (0.07 * 100 = 7.000000000000001 gives 8); the masked ids are the top_k of the mask
 *   noise u0 (descending, ties to the smaller id: SimMIM's order and mim_mask's kernel).  k == 0 (the reference's mean over no rows
 *   is NaN) and k > n are refused.
 *   Draws: one Philox4x32-10 block per (image, position) with vb_forward_mim's key, counter (j, b, d_lo, d_hi) and per-call d;
 *   words 0-3 are the mask noise, the random-patch coin, the random patch id and the replace coin (mpp.py:178-196), in that order,
 *   also when random_patch_prob == 0 (the reference then draws only the mask and the replace coin).  u = (word >> 8) 2^-24; the
 *   random id is (uint64(word 2) n) >> 32; a coin is u < p in float32, p the double rounded to float32.  The random-patch coin's
 *   p is random_patch_prob / (1 - replace_prob), drawn only when random_patch_prob > 0 (replace_prob == 1 is then refused, the
 *   reference's ZeroDivisionError).
 *   Corruption, per masked position j (the reading of mpp.py:188-197 this engine takes): where the random-patch coin is true the
 *   pixels of the ORIGINAL patch at the random id (line 191 reads randomized_input before any write); then, where the replace coin
 *   is true, mask_token (the mask token wins).  Read literally the reference does neither: under TF 2 `.numpy()` returns a copy, so
 *   the writes at 192 and 197 are lost and the encoder sees the clean image; were they views, line 196's int32 cast would index
 *   the batch axis with the 0 / 1 mask, overwrite all of images 0 and 1 with the token, and raise IndexError at batch 1.
 *   Encoder (mpp.py:199-212): row 1 + j = patch.kernel . (corrupted patch j) + patch.bias + pos_embedding[1 + j], row 0 = cls_token +
 *   pos_embedding[0], the encoder's layers over the n + 1 rows.
 *   Head and loss (mpp.py:108-131, 213-216): logits = to_bits(the encoded rows of the masked ids, ascending), K = 2^(bits channels)
 *   classes.  softmax_cross_entropy_with_logits(labels=logits, logits=target [M, 1]) broadcasts the [M, 1] operand to [M, K]
 *   before its softmax, which is then 1 / K everywhere, so loss = ln(K) * mean over the M = batch k masked rows of sum_c
 *   logits[row, c]: the targets, clipping, bucketing, max_pixel_val, mean and std do not reach it.  Summed in double in a fixed
 *   order over the logits as returned. */
typedef struct vb_mpp_config {
  vb_mim_config mim;              /* mim.struct_size = sizeof(vb_mpp_config); masking_ratio and the decoder fields unused */
  double mask_prob;               /* k = ceil(mask_prob * n) */
  double replace_prob;            /* the mask-token coin's probability */
  double random_patch_prob;       /* the random-patch coin's probability is random_patch_prob / (1 - replace_prob) */
  int32_t output_channel_bits;    /* K = 2^(output_channel_bits * channels) <= 2^16; channels must be 3 */
} vb_mpp_config;

/* MPP.__init__: vb_create_mim with encoder->kind VB_KIND_MPP and `mim` pointing at a vb_mpp_config.  Weights: the encoder ViT's
 * names WITH cls_token and without head_norm.* / head.* -- pos_embedding [1, n_p + 1, dim], cls_token [1, 1, dim], patch.kernel
 * [patch_dim, dim] / .bias, layers.L.* -- plus mask_token [patch_dim] (pixel space) and to_bits.kernel [dim, K] / .bias [K]. */

/* One MPP call: img as in vb_forward_mim; loss: one float; logits float32 [batch, k, K] (the masked rows, ids ascending),
 * mask_ids int32 [batch, k] (ascending), source int32 [batch, n] (j for an unchanged position, the random patch id for a
 * random-patch one, -1 for the mask token); the three arrays may be NULL; all outputs in out_mem memory.  Graph capture and replay,
 * the seed (vb_mim_set_seed) and the draw counter as vb_forward_mim's.  Refused: sides not divisible by the patch, more than n_p or
 * VB_MIM_MAX_PATCHES patches, k == 0 or k > n, replace_prob == 1 with random_patch_prob > 0. */
VB_API int vb_forward_mpp(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w, float* loss,
                          float* logits, int32_t* mask_ids, int32_t* source, int32_t out_mem, void* stream);
/* MPP's draws on their own (mim_mask descending, then the corruption draws) for the key `seed` and draw counter `counter`:
 * mask_ids int32 [B, k] ascending and source int32 [B, n] (host).  1 <= k <= n <= VB_MIM_MAX_PATCHES. */
VB_API int vb_op_mpp_draws(int32_t B, int32_t n, int32_t k, double replace_prob, double random_patch_prob, uint64_t seed, uint64_t counter,
                           int32_t* mask_ids, int32_t* source);

/* DistillWrapper (distill.py:87-134), appended within ABI 7: inference semantics and the loss value of the soft branch.
 *   call([img, labels], T, alpha) = ce * (1 - alpha) + distill_loss * alpha, a float32 vector [b], with
 *   ce[i] = categorical_crossentropy(labels[i], student_logits[i], from_logits=True) = sum_c labels[i, c] (lse(s_i) - s_i[c]), the
 *   labels used as given (one-hot or any soft rows, not renormalised), and the distillation term read as Keras computes it:
 *   KLDivergence(y_true, y_pred) clips BOTH arguments to [1e-7, 1].  Here y_pred = log_softmax(distill_logits / T) is <= 0, so it
 *   always clips to 1e-7 and the term never reads the student: per image q[j] = sum_c y'[j, c] (ln y'[j, c] - ln 1e-7) with
 *   y' = clip(softmax(teacher_logits[j] / T), 1e-7, 1) (the clip applied to the float32 softmax, at 1e-7f), and
 *       out[i] = (1 - alpha) ce[i] + alpha T^2 (1 / b) sum_j q[j].
 *   The distillation token still reaches the loss through student_logits; distill_logits and distill_mlp's weights do not (for
 *   finite logits).  This reading comes from Keras' source; the numpy stand-in of the tests clips the same way, and the unmodified
 *   reference DistillWrapper over it returns this vector.  It has not been checked against TensorFlow itself.
 *   hard=True cannot run in the reference: tf.argmax gives [b] integer labels, which categorical_crossentropy refuses against the
 *   [b, K] logits (ValueError "Shapes (b,) and (b, K) are incompatible") at every batch size.  The host class raises that error;
 *   the engine implements no hard distillation.  T == 0 (inf / NaN in the reference) is refused.
 *   Per image, ce and q are sums in double over max-subtracted softmaxes (logits of magnitude ~100 do not overflow); the mean of q
 *   is vb_forward_mim's fixed-order reduction, so eager, captured and replayed calls give the same bits.
 * vb_create_distill: `student` is the student's own vb_config (kind VB_KIND_VIT or VB_KIND_T2T_VIT; a T2TViT of depth 0, built for
 * an injected transformer, is refused: its call is composed on the host).  Weights: the student's names (SURVEY.md App. B) plus
 *   distillation_token [1, 1, dim], distill_mlp.0.gamma / .beta [dim] (the LayerNormalization, eps 1e-3),
 *   distill_mlp.1.kernel [dim, num_classes] / .bias [num_classes] (the Dense).
 * The handle is a student handle: vb_forward and vb_forward_distill run on it as on the student's. */
VB_API int vb_create_distill(const vb_config* student, int device, vb_handle** out);
/* One DistillWrapper call.  img as in vb_forward (img_mem); labels float32 [batch, num_classes] and teacher_logits float32
 * [batch, num_classes] in in_mem memory.  Exactly one of `teacher` (a classifier handle on the same device with num_classes
 * classes) and `teacher_logits` is given.  With a teacher handle the image is uploaded once and the teacher runs through its
 * own vb_forward on `stream`, under its own graph rules, into a buffer of this handle; it is not part of this handle's graph.
 * Then the student with the handle's distillation token (vb_forward_distill's semantics), distill_mlp on the token's row and the
 * loss are captured and replayed under vb_forward's rules, keyed also by the labels and teacher-logit pointers and the bit
 * patterns of temperature and alpha.  Outputs in out_mem memory: loss float32 [batch]; student_logits, distill_logits and
 * teacher_logits_out [batch, num_classes] when not NULL. */
VB_API int vb_forward_distill_loss(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                                   const float* labels, vb_handle* teacher, const float* teacher_logits, int32_t in_mem,
                                   double temperature, double alpha, float* loss, float* student_logits, float* distill_logits,
                                   float* teacher_logits_out, int32_t out_mem, void* stream);
/* The loss kernels of vb_forward_distill_loss on their own, over host buffers: student_logits, labels, teacher_logits float32
 * [B, K] -> out float32 [B].  T == 0 is refused. */
VB_API int vb_op_distill_loss(const float* student_logits, const float* labels, const float* teacher_logits, int32_t B, int32_t K,
                              double temperature, double alpha, float* out);

/* Row softmax of fp32 scores into bf16 probabilities (the T2T attention): p[r, j] = softmax_j(s[r, j] * scale) for j < n,
 * p[r, n..npad) = 0.  s [rows, lds], p [rows, ldp] (uploaded and downloaded whole); n <= npad <= ldp. */
VB_API int vb_op_softmax_rows(const float* s, int32_t lds, float* p, int32_t ldp, int32_t rows, int32_t n, int32_t npad, float scale,
                              int32_t iters, float* elapsed_ms);

#ifdef __cplusplus
}
#endif
#endif /* VITB200_H_ */
