// DistillWrapper's loss (distill.py:108-134, soft branch) on the device: one CTA per image reads that image's student logits,
// labels and teacher logits and writes its cross-entropy and its KL term, the existing fixed-order reduction averages the KL
// terms, and a last pass combines them.  See kernels.cuh for the contract and include/vitb200.h for the reading of the KL term.
#include "kernels.cuh"

namespace vb {
namespace {

constexpr int DISTILL_THREADS = 256;

// A fixed tree over the CTA: the same bits on every call.  red holds DISTILL_THREADS values; the result is broadcast.
template <typename V, typename Op>
__device__ V distill_block_reduce(V v, V* red, Op op) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int s = DISTILL_THREADS / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = op(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  const V r = red[0];
  __syncthreads();                                           // red is reused by the next reduction
  return r;
}

// Image b: ce[b] = sum_c y[c] (lse(s) - s[c]) (categorical_crossentropy from logits, labels as given) and
// q[b] = sum_c y'[c] (ln y'[c] - ln 1e-7f), y' = clip(float32(softmax(t / T)), 1e-7f, 1) (KLDivergence with y_pred clipped to
// 1e-7f, see vitb200.h).  Both softmaxes subtract the row maximum; the sums run in double.
__global__ void __launch_bounds__(DISTILL_THREADS)
distill_rows_kernel(const float* __restrict__ S, const float* __restrict__ Y, const float* __restrict__ Tl, int K, double inv_T,
                    double* __restrict__ ce, double* __restrict__ q) {
  __shared__ double red[DISTILL_THREADS];
  const size_t off = static_cast<size_t>(blockIdx.x) * K;
  const float* s = S + off;
  const float* y = Y + off;
  const float* t = Tl + off;
  auto dmax = [](double a, double b) { return a > b ? a : b; };
  auto dadd = [](double a, double b) { return a + b; };
  double ms = -INFINITY, mt = -INFINITY;
  for (int c = threadIdx.x; c < K; c += DISTILL_THREADS) {
    ms = dmax(ms, static_cast<double>(s[c]));
    mt = dmax(mt, static_cast<double>(t[c]) * inv_T);
  }
  ms = distill_block_reduce(ms, red, dmax);
  mt = distill_block_reduce(mt, red, dmax);
  double zs = 0.0, zt = 0.0;
  for (int c = threadIdx.x; c < K; c += DISTILL_THREADS) {
    zs += exp(static_cast<double>(s[c]) - ms);
    zt += exp(static_cast<double>(t[c]) * inv_T - mt);
  }
  zs = distill_block_reduce(zs, red, dadd);
  zt = distill_block_reduce(zt, red, dadd);
  const double ls = log(zs), inv_zt = 1.0 / zt, ln_eps = log(static_cast<double>(1e-7f));
  // ce = sum_c y (ms - s) + ls sum_c y: both sums are of non-negative terms for non-negative labels, so no cancellation
  double gap = 0.0, ysum = 0.0, kl = 0.0;
  for (int c = threadIdx.x; c < K; c += DISTILL_THREADS) {
    const double yc = static_cast<double>(y[c]), sc = static_cast<double>(s[c]);
    gap += yc * (ms - sc);
    ysum += yc;
    const float p = fminf(fmaxf(static_cast<float>(exp(static_cast<double>(t[c]) * inv_T - mt) * inv_zt), 1e-7f), 1.0f);
    kl += static_cast<double>(p) * (log(static_cast<double>(p)) - ln_eps);
  }
  gap = distill_block_reduce(gap, red, dadd);
  ysum = distill_block_reduce(ysum, red, dadd);
  kl = distill_block_reduce(kl, red, dadd);
  if (threadIdx.x == 0) {
    ce[blockIdx.x] = gap + ls * ysum;
    q[blockIdx.x] = kl;
  }
}

// out[b] = (1 - alpha) ce[b] + dterm, dterm = alpha T^2 mean(q) (one float written by the reduction)
__global__ void distill_out_kernel(const double* __restrict__ ce, const float* __restrict__ dterm, double one_minus_alpha, int B,
                                   float* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b < B) out[b] = static_cast<float>(one_minus_alpha * ce[b] + static_cast<double>(*dterm));
}

}  // namespace

void distill_loss(const float* student_logits, const float* labels, const float* teacher_logits, int B, int K, double T, double alpha,
                  double* ce, double* q, float* dterm, float* out, cudaStream_t s) {
  VB_CHECK(B >= 1 && K >= 1, "distill_loss: bad shape");
  VB_CHECK(T != 0.0, "DistillWrapper: temperature 0 divides the logits by zero");
  distill_rows_kernel<<<B, DISTILL_THREADS, 0, s>>>(student_logits, labels, teacher_logits, K, 1.0 / T, ce, q);
  VB_CUDA(cudaGetLastError());
  count_launch();
  mim_loss_final(q, B, alpha * T * T / static_cast<double>(B), dterm, s);   // distill.py:126-129: sum / b, then * T^2
  distill_out_kernel<<<(B + 255) / 256, 256, 0, s>>>(ce, dterm, 1.0 - alpha, B, out);
  VB_CUDA(cudaGetLastError());
  count_launch();
}

}  // namespace vb
