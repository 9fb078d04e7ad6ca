"""Error of the erf approximations used by the fc1 GELU epilogue (csrc/gemm_wgmma.cu), against scipy's erf,
in absolute terms and in bf16 ulps of the GELU output.  Runs on CPU."""
import numpy as np
from scipy.special import erf

x = np.linspace(-10, 10, 4000001)
g = 0.5 * x * (1 + erf(x / np.sqrt(2)))
ulp = np.maximum(np.abs(g), 1e-30) * 2.0 ** -8
z = np.abs(x) / np.sqrt(2)


def report(name, erf_abs):
    ga = 0.5 * x + 0.5 * np.abs(x) * erf_abs
    d = np.abs(ga - g)
    print(f"{name:34s} max abs err {d.max():.3e}   max err in bf16 ulps (|gelu| > 0.05) {(d / ulp)[np.abs(g) > 0.05].max():.4f}")




def fit_tail(deg=5, amax=6.0):
    """Weighted (iteratively re-weighted least squares ~ minimax) fit of q(a) = log2(erfc(a/sqrt2)/2), q(0) = -1."""
    from scipy.special import erfc
    a = np.cos(np.pi * (np.arange(4000) + 0.5) / 4000) * amax / 2 + amax / 2
    target = np.log2(0.5 * erfc(a / np.sqrt(2)))
    w = a * 2.0 ** target + 1e-6                      # d gelu = |x| 2^q ln2 dq
    V = np.vander(a, deg + 1, increasing=True)
    for _ in range(30):
        c, *_ = np.linalg.lstsq(V[:, 1:] * w[:, None], (target + 1) * w, rcond=None)
        err = a * (2.0 ** (-1 + V[:, 1:] @ c) - 2.0 ** target)
        w = w * (1 + 0.5 * np.abs(err) / np.abs(err).max())
    return np.concatenate([[-1.0], c]).astype(np.float32)


c = fit_tail()
print("tail polynomial q(a), a = |x| (gemm_wgmma.cu uses -a, odd terms negated):", [f"{float(v):.9e}" for v in c])
xa = np.minimum(np.abs(x), 6.0).astype(np.float32)
q = np.full_like(xa, c[-1])
for k in range(len(c) - 2, -1, -1):
    q = q * xa + c[k]
d = np.abs((np.maximum(x, 0) - xa * np.exp2(q)) - g)
print(f"{'2^poly5 tail (the kernel)':34s} max abs err {d.max():.3e}   max err in bf16 ulps (|gelu| > 0.05) {(d / ulp)[np.abs(g) > 0.05].max():.4f}")

t = 1 / (1 + 0.3275911 * z)
report("A-S 7.1.26 (previous kernel)", 1 - (((((1.061405429 * t - 1.453152027) * t) + 1.421413741) * t - 0.284496736) * t + 0.254829592) * t * np.exp(-z * z))
p = 1 + z * (0.0705230784 + z * (0.0422820123 + z * (0.0092705272 + z * (0.0001520143 + z * (0.0002765672 + z * 0.0000430638)))))
report("A-S 7.1.28", 1 - 1 / p ** 16)
t = 1 / (1 + 0.47047 * z)
report("A-S 7.1.25", 1 - (0.3480242 * t - 0.0958798 * t ** 2 + 0.7478556 * t ** 3) * np.exp(-z * z))
gt = 0.5 * x * (1 + np.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))
d = np.abs(gt - g)
print(f"{'tanh GELU (NOT used: approximate)':34s} max abs err {d.max():.3e}   max err in bf16 ulps (|gelu| > 0.05) {(d / ulp)[np.abs(g) > 0.05].max():.4f}")
