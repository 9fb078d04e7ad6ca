// Launch interfaces of the non-tensor-core kernels (kernels.cu).  T is float (exact-fp32 gate path) or
// __nv_bfloat16 (activations of the tensor-core path); all reductions / statistics are fp32.
#pragma once
#include "common.h"

namespace vb {

// im2col for non-overlapping patches: 'b (h p1) (w p2) c -> b (h w) (p1 p2 c)' (vit.py:142).
// img NHWC fp32 [B,H,W,C] -> out [B*(cls_row + gh*gw), ldo], columns [0, ph*pw*C) filled, [.., ldo) zeroed;
// when cls_row == 1 the first row of every image is all zeros (its value comes from the GEMM epilogue).
template <typename T>
void im2col(const float* img, T* out, int B, int H, int W, int C, int ph, int pw, int cls_row, int ldo, cudaStream_t s);

// R[b*rows + t, :] = pos[t, :] (+ cls - bias on t == 0 when has_cls): the additive term of the patch-embedding
// GEMM epilogue that realises cls-token concat + pos_embedding add (vit.py:163-165, cait.py:184).
template <typename T>
void build_embed_residual(T* R, const float* pos, const float* cls, const float* bias, int B, int rows, int dim,
                          int has_cls, cudaStream_t s);

// LayerNorm over the last axis (biased variance; Keras eps 1e-3, vit.py:18; CvT's own LayerNorm eps 1e-5, cvt.py:30-43).
// x [M, ldx] -> out [M, ldo].  pad_to > D: columns [D, pad_to) of every output row are zeroed (pitch-padded token rows feeding a
// K-padded GEMM).
template <typename T>
void layernorm(const T* x, int ldx, const float* gamma, const float* beta, T* out, int ldo, int M, int D, cudaStream_t s, int pad_to = 0,
               float eps = 1e-3f);

// Row softmax of materialised fp32 scores -> bf16 probabilities: P[r, j] = softmax_j(S[r, j] * scale), j < n; P[r, n..npad) = 0.
// scale_log2 = scale * log2(e).  Rows of up to 4096 keys stay in registers; longer rows take a three-pass kernel.
void softmax_rows_bf16(const float* S, int lds, __nv_bfloat16* P, int ldp, long long rows, int n, int npad, float scale_log2, cudaStream_t s);
// out[b, c, j] = in[b, j, c] for c < cols, j < n; out[b, c, n..npad) = 0 (bf16; batch pitches in elements)
void transpose_rows_bf16(const __nv_bfloat16* in, int ldi, long long in_batch, __nv_bfloat16* out, int ldo, long long out_batch, int B,
                         int n, int npad, int cols, cudaStream_t s);

// out[M,N] (TO) = epi(A[M,K] (TA, lda) x W), W element (k,n) at W[k*wsk + n*wsn]; fp32 FMA accumulation.
// epi = (+bias) -> act (Act: GELU(erf) / hard-swish / SiLU) -> (*scale) -> (+res[m*ldr + n]).
template <typename TA, typename TW, typename TO>
void gemm_simt(const TA* A, int lda, const TW* W, int wsk, int wsn, TO* out, int ldc, int M, int N, int K,
               const float* bias, const float* scale, const TO* res, int ldr, int act, cudaStream_t s);

// Generic attention through materialised scores (any n, d, variant), S fp32 [B,h,nq,nk] workspace.
// q: [B, nq, *] rows of pitch ldq with head hh at columns [hh*dh, (hh+1)*dh); k, v likewise (nk rows per batch).
template <typename T>
void attn_scores(const T* q, int ldq, const T* k, int ldk, float* S, int B, int heads, int nq, int nk, int dh, float scale,
                 cudaStream_t s);
// In-place head mix: S[b,g,i,j] = sum_h S[b,h,i,j] * Wmix[h,g]; optional LayerNorm over g (gamma/beta [heads]).
void attn_head_mix(float* S, const float* Wmix, const float* gamma, const float* beta, int B, int heads, int nq, int nk,
                   cudaStream_t s);
void attn_softmax(float* S, long long rows, int nk, cudaStream_t s);
// gelu_out: exact-erf GELU of every output element (PosBias::gelu_out)
template <typename T>
void attn_pv(const float* S, const T* v, int ldv, T* out, int ldo, int B, int heads, int nq, int nk, int dh, cudaStream_t s,
             int gelu_out = 0);
// S[b,h,i,j] += the relative-position bias of (i, j) (PosBias, common.h); S fp32 [B,h,nq,nk]
void attn_pos_bias(float* S, const PosBias& pb, int B, int heads, int nq, int nk, cudaStream_t s);

// The strided pixels of a map (LeViT's stride-2 1x1 VALID query convolution, levit.py:75): in [B, H, W, C] rows of pitch ldi ->
// out [B, ceil(H/step) * ceil(W/step), C] rows of pitch ldo, out pixel (r, c) = in pixel (step*r, step*c).
template <typename T>
void gather_grid(const T* in, int ldi, T* out, int ldo, int B, int H, int W, int C, int step, cudaStream_t s);

// CvT's attention projections up to the pointwise convolutions (cvt.py:79-92,103-104), both depthwise convolutions of a block
// from one read of the input (kv == null: the q map only, Twins-SVT's PEG with its residual folded into the centre tap): q = dw_q(y) (stride 1) and kv = dw_kv(y) (stride kv_stride: 1 or 2), k x k (k <= 7), TF SAME
// padding (total max((out - 1) * stride + k - in, 0), the smaller half first), then + a per-channel shift.
//   x [B*H*W, ldx] NHWC rows; y = LN(x) when stats != null: the rows' (sum, sumsq) partials [C/64][B*H*W] (the GEMM epilogue's
//   stats_out format) over D true columns with eps, times gamma plus beta ([C], zero on pad channels); y = x when stats == null.
//   The padding is zeros of y.  wq / wkv: taps [k*k][C] (row-major window, BatchNorm scale folded in), bq / bkv: shifts [C].
//   q [B*H*W, ldq], kv [B*ceil(H/s)*ceil(W/s), ldkv]: columns [0, C) written.
template <typename T>
void dwconv_qkv(const T* x, int ldx, const float* stats, const float* gamma, const float* beta, int D, float eps, const float* wq,
                const float* bq, T* q, int ldq, const float* wkv, const float* bkv, T* kv, int ldkv, int B, int H, int W, int C, int k,
                int kv_stride, cudaStream_t s);

// MobileViT's MV2 depthwise step (mobile_vit.py:142-145,157-160): a 3 x 3 depthwise convolution with stride 1 or 2 and TF SAME
// padding (total max((out - 1) * stride + 3 - in, 0), the smaller half first), its BatchNorm folded into the taps and a shift,
// then SiLU on store.  x [B*H*W, ldx] NHWC rows -> out [B*ceil(H/s)*ceil(W/s), ldo]; w: taps [9][Cp] (row-major window), shift
// [Cp], both zero on channels >= C; columns [C, Cp) of out are written as zero.  bf16: 8 channels per thread in 16-byte
// accesses (Cp, ldx, ldo multiples of 8); fp32: one channel per thread.
template <typename T>
void dwconv_bn_act(const T* x, int ldx, const float* w, const float* shift, T* out, int ldo, int B, int H, int W, int C, int Cp, int stride,
                   cudaStream_t s);

// z[b,:] = LN(pool(X[b]))  with pool = row 0 (cls) or mean over the n rows; fp32 out [B, D].  gamma == null: no LayerNorm.
template <typename T>
void pool_layernorm(const T* X, int n, int ldx, const float* gamma, const float* beta, float* out, int B, int D, int mean_pool,
                    cudaStream_t s);

// dst[b, doff + t, :] = src[b, soff + t, :], t < count  (token concat / slicing; batch pitches in rows).
template <typename T>
void copy_tokens(const T* src, int src_rows, int soff, T* dst, int dst_rows, int doff, int count, int B, int D, cudaStream_t s);
// dst[b, 0, :] = vec (fp32) for every b (cls token broadcast, cait.py:189).
template <typename T>
void broadcast_row(const float* vec, T* dst, int dst_rows, int B, int D, cudaStream_t s);

// dst[b, t, :] = vec[t, :] (fp32 [nt, D]) for every b (PatchMerger queries, vit_with_patch_merger.py:47,51).
template <typename T>
void broadcast_rows(const float* vec, T* dst, int B, int nt, int D, cudaStream_t s);

// T2T soft split (t2t.py:43-44): tf.image.extract_patches(sizes k, strides `stride`, rates 1, padding SAME) +
// 'b h w c -> b (h w) c'.  in [B,H,W,C] (image or token map) -> out [B*(cls_row + oh*ow), ldo], oh = ceil(H/stride);
// columns [0, k*k*C) hold the patch vector ((k_row, k_col, c), c fastest), [.., ldo) and the optional cls row are zero.
// ldi: pitch of one input pixel's channel vector (0 = C).  mode (may be null): see UnfoldMode.
// Twins-SVT's global to_kv (twins_svt.py:168,180), Conv2D(k, stride k, VALID) of the PreNorm LayerNorm of the map: `valid` takes
// floor((H - k) / stride) + 1 windows per side with no padding, and `stats` applies the LayerNorm on load from the pixels' (sum,
// sumsq) partials [C_pitch/64][B*H*W] (the GEMM epilogue's stats_out format) over d true channels with eps, times gamma plus beta.
// A folded LayerNorm cannot serve this GEMM: one patch row spans k^2 pixels with different statistics.  `gelu`: the exact-erf
// GELU of every loaded value, after the LayerNorm when there is one (RegionViT's 3-conv local tokenizer, regionvit.py:211-218);
// padded taps stay zero.
struct UnfoldMode {
  bool valid = false;
  const float* stats = nullptr;
  int parts = 0, d = 0;
  float eps = 1e-5f;
  const float *gamma = nullptr, *beta = nullptr;
  bool gelu = false;
};
template <typename TI, typename TO>
void unfold_same(const TI* in, TO* out, int B, int H, int W, int C, int k, int stride, int cls_row, int ldo, cudaStream_t s, int ldi = 0,
                 const UnfoldMode* mode = nullptr);

// Rows of a pixel-major map <-> window-major order (the fallback of the windowed attention, common.h Window): window-major row
// t = bw * p^2 + i is the map's row win.row(bw, i).  to_window: out[t] = in[win.row(t)]; else out[win.row(t)] = in[t].  `cols`
// columns of `rows` = (number of windows) * p^2 rows.
template <typename T>
void window_rows(const T* in, int ldi, T* out, int ldo, int cols, const Window& win, long long rows, bool to_window, cudaStream_t s);
// The same for RegionViT's regional-to-local windows (the fallback of attention_r2l): window-major row t = bw * n + i, n = 1 +
// p * width(), is the regional row reg_row0 + bw for i == 0 and the map's row win.row(bw, i - 1) otherwise; win.count windows.
template <typename T>
void r2l_rows(const T* in, int ldi, T* out, int ldo, int cols, const Window& win, long long reg_row0, bool to_window, cudaStream_t s);

// CCT tokenizer tail (cct.py:196-200,213): ReLU -> MaxPool2D(k, stride, padding 'SAME') -> 'b h w c -> b (h w) c', NHWC.
// in [B, H, W, C] -> out [B, rows, C], oh = ceil(H / stride), rows >= oh * ow; total padding max((oh-1)*stride + k - H, 0) with
// the smaller half first, padded taps never win the max.  ReLU is applied after the max (both are monotone: the same value).
// pos (fp32 [oh*ow, C], may be null) is added after the ReLU; rows [oh*ow, rows) are zero (the 'none' embedding's zero padding).
template <typename T>
void maxpool_relu_same(const T* in, T* out, int B, int H, int W, int C, int k, int stride, const float* pos, int rows, cudaStream_t s);

// NesT's aggregation tail and position add (nest.py:111-123,140-142), NHWC rows: in [B*H*W, ldi] -> out [B*oh*ow, ldo].
//   ln (may be null): LayerNorm each input pixel on load from its (sum, sumsq) partials [parts][B*H*W] (the GEMM epilogue's
//     stats_out format) over d true channels with eps, times gamma plus beta; the fp32 engine passes null after its own LayerNorm.
//   pool: MaxPool2D(3, 2, 'SAME'), oh = ceil(H / 2), total padding max((oh - 1) * 2 + 3 - H, 0) with the smaller half first, and
//     padded taps never win; !pool: oh = H, each pixel as it is (in may equal out).
//   pos (may be null): the next Transformer's scalar pos[(y % bh) * bw + x % bw] added to the C true channels of output pixel
//     (y, x) of bh x bw blocks; columns [C, ldo) are written as zero.
//   stats_out (may be null; ldo % 64 == 0): the stored rows' (sum, sumsq) partials [ldo/64][B*oh*ow].
struct NestPoolLn {
  const float* stats = nullptr;
  int parts = 0, d = 0;
  float eps = 1e-5f;
  const float *gamma = nullptr, *beta = nullptr;
};
template <typename T>
void nest_pool(const T* in, int ldi, const NestPoolLn* ln, int B, int H, int W, int C, bool pool, const float* pos, int bh, int bw,
               T* out, int ldo, float* stats_out, cudaStream_t s);

// CCT sequence pooling (cct.py:291-299): per image b, y_t = LayerNorm(X[b, t]) (eps 1e-3), w_t = softmax_t(y_t . pw + pb),
// z[b] = sum_t w_t y_t.  X [B, n, D] -> z fp32 [B, D]; D <= 1024.  One CTA per image, fp32 statistics, online softmax.
template <typename T>
void seq_pool(const T* X, int n, int D, const float* gamma, const float* beta, const float* pw, const float* pb, float* z, int B,
              cudaStream_t s);

// out[r, 0:cols] = in[r, 0:cols], out[r, cols:ldo] = 0 (type conversion with a row-pitch change).
template <typename TI, typename TO>
void convert_rows(const TI* in, int ldi, TO* out, int ldo, long long rows, int cols, cudaStream_t s);

template <typename TI, typename TO>
void convert(const TI* in, TO* out, long long count, cudaStream_t s);
void add_inplace_f32(float* a, const float* b, long long count, cudaStream_t s);
// Wt[n*ldw + k] = bf16(W[k*N + n]) : Keras [K,N] fp32 -> K-major bf16 rows (zero padded to ldw)
// row_scale (may be null): Wt[n*ldw + k] = bf16(W[k*N + n] * row_scale[k])  (LayerNorm gamma folded into the weight)
void pack_weight_bf16(const float* W, __nv_bfloat16* Wt, int K, int N, int ldw, cudaStream_t s, const float* row_scale = nullptr);
// Head-padded copy of a Dense kernel (fp32, Keras [K, N] layout) for layers whose dim_head is widened to the attention
// kernel's head width with zero weights.  pad_rows == 0: the N = groups*heads*dh output columns [g][h][d] become
// groups*heads*dhp columns, column (g, h, d >= dh) = 0 (to_qkv: groups 3, to_q: 1, to_kv: 2).  pad_rows == 1: the
// K = heads*dh input rows become heads*dhp rows, row (h, d >= dh) = 0 (to_out).  `other` is the untouched dimension.
void pad_heads_f32(const float* W, float* Wp, int other, int groups, int heads, int dh, int dhp, int pad_rows, cudaStream_t s);
// Constants of a LayerNorm folded into the following Dense (see gemm_wgmma.cu):
//   c1[n] = sum_k float(Wt[n,k])   (the gamma-scaled, bf16-rounded weights the tensor core really multiplies)
//   c2[n] = sum_k beta[k] * W[k,n] + (bias ? bias[n] : 0)
void ln_fold_consts(const float* W, const __nv_bfloat16* Wt, int ldw, const float* beta, const float* bias, float* c1, float* c2,
                    int K, int N, cudaStream_t s);
// stats[c, m] = (sum, sum of squares) of X[m, 64c .. 64c+63]  ([D/64][M] float2: the format the GEMM epilogue emits and the
// LayerNorm-folded GEMM's statistics warp reduces); D % 64 == 0.  pitch > 0: stats[c * pitch + m] instead, for rows that are
// the tail of a longer statistics buffer (RegionViT's regional rows after the local ones).
void row_stats_bf16(const __nv_bfloat16* X, int ldx, float* stats, int M, int D, cudaStream_t s, long long pitch = 0);

// ---- adaptive token sampling (ATS-ViT, ats_vit.py:77-132, 191-258; ats.cu).  Image b's rows sit at pitch P as [cls, its
// c_b kept tokens in ascending id order, dead rows]; rows[b] = c_b + 1 (the live rows: the key count of its masked attention),
// and C (one int on the device) is the batch maximum of the c_b.
constexpr int ATS_MAX_DH = 256;          // widest head ats_sample reads
constexpr int ATS_MAX_TOKENS = 65536;    // the noise counter holds the column in 16 bits: patches + 1 <= 65,536
// rows[b] = P, *C = P - 1, ids[b, t] = t
void ats_init(int* rows, int* C, int* ids, int B, int P, cudaStream_t s);
// One CTA per image.  When *C <= K the layer keeps every row: sel[b, t] = t for t < rows[b], rows_new = rows.  Otherwise,
// from the fused q | k | v rows (head h at columns h*dh, HD + h*dh, 2 HD + h*dh; dh the stored width, pad columns zero): the cls
// query's softmax over its valid keys 0..c (fp32, `scale`), weighted by the value norms and summed over heads, normalised and
// logged; then K Gumbel-max draws with u = (Philox4x32-10 word 0 >> 8) * 2^-24, key rng[0], counter (j | k << 16, b, rng[1]),
// j = C - c + i - 1 for compact token i.  draws[b, k] = the winner's position in the reference's left-padded layout (argmax + 1);
// sel[b, 0 .. rows_new[b]) = 0 then the distinct winners in ascending order.  scratch: 3 * B * P floats.
template <typename T>
void ats_sample(const T* qkv, int ld, int B, int P, int heads, int dh, float scale, const int* rows, const int* C, int K,
                const unsigned long long* rng, float* scratch, int* sel, int Pn, int* rows_new, int* draws, cudaStream_t s);
// Xn [B * Pn, dim] = the rows sel picks from X [B * P, dim] (zero rows from rows_new[b] on), ids_n likewise from ids (0 on dead
// rows); *C_new = max(rows_new) - 1; rng[1] += 1 when *C_old > K (the layer sampled).
template <typename T>
void ats_gather(const T* X, int P, T* Xn, int Pn, int dim, const int* sel, const int* rows_new, const int* ids, int* ids_n, int B,
                const int* C_old, int K, int* C_new, unsigned long long* rng, cudaStream_t s);
// out [B, P - 1] = the reference's returned token ids (ats_vit.py:315): image b's kept patch ids in columns [C - c_b, C), -1 elsewhere
void ats_ids_out(const int* ids, int P, const int* rows, const int* C, int* out, int B, cudaStream_t s);
// attn_softmax with the keys j >= nk_img[row / rows_per_img] of every row masked (nk_img may be null: none), and with
// diag_nq > 0 also the key j == row % diag_nq (locality self-attention's diagonal, rows [.., nq] with nq == diag_nq == nk): their
// weight is exactly 0
void attn_softmax_masked(float* S, long long rows, int nk, long long rows_per_img, const int* nk_img, cudaStream_t s, int diag_nq = 0);

// ---- shifted patch tokens (vit_for_small_dataset.py:15-47, 142-157; small_vit.cu).  out [B * (1 + np), ldo]: per image a zero
// cls row, then patch t = (gy, gx) of the (H / p) x (W / p) grid as the vector [p1][p2][view][c] of the image concatenated with
// its four one-pixel shifts (view 1: x[:, w - 1], 2: x[:, w + 1], 3: x[h - 1], 4: x[h + 1], zero past the edge), so element
// ((p1 p + p2) 5 + view) C + c; columns from 5 C p^2 to ldo are zero.  img fp32 NHWC [B, H, W, C].
template <typename T>
void spt_rows(const float* img, T* out, int B, int H, int W, int C, int p, int ldo, cudaStream_t s);

// ---- masked image modelling (MAE, mae.py:49-92; SimMIM, simmim.py:82-129; mim.cu).  idx [B, n] holds each image's noise
// permutation, the masked patch ids first: MAE's argsort of u ascending (ties to the smaller id), SimMIM's top_k order (u
// descending, ties to the smaller id).
constexpr int MIM_MAX_PATCHES = 4096;    // patches per image the mask kernel sorts in shared memory
// One CTA per image: u[b, j] = (Philox4x32-10 word 0 >> 8) * 2^-24, key rng[0], counter (j, b, rng[1] low, rng[1] high), sorted
// into idx (descending != 0: SimMIM's order).  rng[1] advances by one per launch; rng[2] is the kernel's CTA-completion counter (0
// between launches).
void mim_mask(int B, int n, int descending, unsigned long long* rng, int* idx, cudaStream_t s);
// out [B * count, ldo]: row b * count + i = the (p1, p2, c) patch vector of id j = idx[b * n + off + i] (idx null: j = i) read from
// the NHWC image, columns [ph pw C, ldo) zero; R (may be null) [B * count, dim]: pos[1 + j] (pos_embedding [np + 1, dim]).
// MPP (cls non-null, idx null, count = n + 1): row 0 of each image is the cls row (zero, R = pos[0] + cls - bias) and row 1 + j
// takes the pixels of patch src[b * n + j], or mask_row [ph pw C] where that is -1, with R = pos[1 + j].
template <typename T>
void mim_patch_rows(const float* img, int B, int H, int W, int C, int ph, int pw, const int* idx, int n, int off, int count, T* out, int ldo,
                    const float* pos, T* R, int dim, cudaStream_t s, const int* src = nullptr, const float* mask_row = nullptr,
                    const float* cls = nullptr, const float* bias = nullptr);
// MPP's corruption draws (mpp.py:181-197) after mim_mask (descending) drew the call's mask into idx: source [B, n] (j, the random
// patch id, or -1 for the mask token) and mask_ids [B, ldm] (the first k ids of idx, ascending), from words 1-3 of the Philox
// block mim_mask used (counter rng[1] - 1).  p_rand = random_patch_prob / (1 - replace_prob); the random-patch coin is drawn only
// when random_patch_prob > 0.
void mpp_draws(int B, int n, int k, const int* idx, const unsigned long long* rng, double random_patch_prob, double p_rand,
               double replace_prob, int* source, int* mask_ids, int ldm, cudaStream_t s);
// *loss = ln(K) * (sum of logits [rows, ldl] over the columns [0, K)) / rows, a fixed-order reduction in double as mim_loss's
// (partial: mim_loss_blocks(rows) doubles)
template <typename T>
void mpp_loss(const T* logits, int ldl, int K, long long rows, double* partial, float* loss, cudaStream_t s);
// Z [B * n, D]: image b's row t < nm = mask_token + dpe[idx[b, t]], row t >= nm = E[b (n - nm) + t - nm] + dpe[idx[b, t]]
template <typename T>
void mim_decoder_rows(const T* E, const int* idx, int B, int n, int nm, const float* mask_token, const float* dpe, T* Z, int D, cudaStream_t s);
// X [B * n, D]: image b's rows idx[b, i], i < nm, replaced by mask_token + pos[1 + idx[b, i]]
template <typename T>
void mim_mask_tokens(T* X, const int* idx, int B, int n, int nm, const float* mask_token, const float* pos, int D, cudaStream_t s);
// out [B * count, D]: row b * count + i = X row b * n + (idx ? idx[b * n + i] : i)
template <typename T>
void mim_take_rows(const T* X, int n, const int* idx, T* out, int B, int count, int D, cudaStream_t s);
// *loss = mean(pred^2) over pred [B * nm, pd] (img null: MAE), or mean(|pred - masked patch|) / nm with the patch of row b nm + i
// read from the image at id idx[b * n + i] (SimMIM).  Two fixed-order passes in double, no atomics: partial holds
// mim_loss_blocks(B * nm) doubles.
int mim_loss_blocks(long long rows);
template <typename T>
void mim_loss(const T* pred, int pd, int B, int nm, const float* img, int H, int W, int C, int ph, int pw, const int* idx, int n,
              double* partial, float* loss, cudaStream_t s);
// *loss = float(scale * (the sum of partial [G])), summed in double by one CTA in a fixed order (the final step of mim_loss)
void mim_loss_final(const double* partial, int G, double scale, float* loss, cudaStream_t s);
// DistillWrapper's soft loss (distill.py:119-134, the reading of include/vitb200.h), B images of K classes, all [B, K] float32 rows
// on the device: ce [B] and q [B] (doubles) get each image's cross-entropy and KL term, *dterm = alpha T^2 mean(q) through
// mim_loss_final, and out [B] = (1 - alpha) ce + dterm.  T == 0 is refused.
void distill_loss(const float* student_logits, const float* labels, const float* teacher_logits, int B, int K, double T, double alpha,
                  double* ce, double* q, float* dterm, float* out, cudaStream_t s);

long long launch_counter();      // number of kernel launches issued through these wrappers (process-wide)
void count_launch(int n = 1);

}  // namespace vb
