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
       VB_KIND_CVT = 9, VB_KIND_TWINS_SVT = 10, VB_KIND_CROSSFORMER = 11 };
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
 * VB_KIND_TWINS_SVT and VB_KIND_CROSSFORMER are refused here: their handles come from vb_create_levit, vb_create_cvt,
 * vb_create_twins_svt and vb_create_crossformer. */
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

/* DistillMixin.call with a distillation token (reference: distill.py:16-45, DistillableViT distill.py:47-58; ViT only):
 * patch embedding + cls + positions, the token appended as the LAST row, the transformer over n + 2 rows, then
 * logits = mlp_head(pool(x[:, :-1])) and distill_out = x[:, -1].
 * distill_token: HOST float32 [dim] (the caller's trainable variable, distill.py:133).  logits [batch, num_classes] and
 * distill_out [batch, dim] live in `out_mem` memory.  img as in vb_forward.
 * LeViT with a distillation head (levit.py:210,220-224): distill_token must be NULL; logits [batch, num_classes] =
 * mlp_head(pool(x)) and distill_out [batch, num_distill_classes] = distill_head(pool(x)). */
VB_API int vb_forward_distill(vb_handle* h, const float* img, int32_t img_mem, int32_t batch, int32_t img_h, int32_t img_w,
                       const float* distill_token, float* logits, float* distill_out, int32_t out_mem, void* stream);

/* ---- the stages of <Model>.call on their own (SURVEY.md 8f f1/f4): the attribute surface the reference's wrappers and the
 * injected-transformer shell use.  ViT / DeepViT / parallel ViT / CaiT / patch-merger ViT / T2TViT; not CrossViT, CCT, LeViT,
 * CvT, Twins-SVT or CrossFormer. */

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
 *   epi     (+bias[N]) -> exact-erf GELU (gelu != 0) -> (*scale[N]) -> (+res[m, n]).  res == out: the residual is the
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

/* Row softmax of fp32 scores into bf16 probabilities (the T2T attention): p[r, j] = softmax_j(s[r, j] * scale) for j < n,
 * p[r, n..npad) = 0.  s [rows, lds], p [rows, ldp] (uploaded and downloaded whole); n <= npad <= ldp. */
VB_API int vb_op_softmax_rows(const float* s, int32_t lds, float* p, int32_t ldp, int32_t rows, int32_t n, int32_t npad, float scale,
                              int32_t iters, float* elapsed_ms);

#ifdef __cplusplus
}
#endif
#endif /* VITB200_H_ */
