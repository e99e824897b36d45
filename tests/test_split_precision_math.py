"""Why the tensor-core contractions run in split precision (SURVEY.md section 7 hard part 4; vbx_mma_kernels.cu,
vbx_project_tc.cu), shown with a bit-level numpy emulation of the operand splits the kernels use:

    tf32(x)    = round-to-nearest of x to 10 explicit mantissa bits        ((bits + 0x1000) & 0xffffe000)
    2-way      : x ~ hi + lo,        hi = tf32(x), lo = tf32(x - hi)              -> products hi*hi' + lo*hi' + hi*lo'
    3-way      : x = x1 + x2 + x3    exactly (11 + 11 + 11 significant bits >= 24) -> six products (front end)

Products of two tf32 numbers are exact in float32 and the tensor core accumulates in float32, so a float32 matmul of the
split parts is a faithful stand-in.  The point: plain TF32 misses the 1e-4 parity bar (log-likelihoods off by ~1e-2,
soft posteriors by ~5e-4, the projection by 3e-4 of its range), the 3xTF32 scheme meets it with more than an order to spare."""
import numpy as np

from vbx_b200 import synth

f32, f64 = np.float32, np.float64


def tf32(x):
    b = np.ascontiguousarray(x, dtype=f32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(f32)


def split2(x):
    hi = tf32(x)
    return hi, tf32(x.astype(f32) - hi)


def split3(x):
    x = x.astype(f32)
    x1 = tf32(x)
    r1 = x - x1                      # exact: the remainder of a rounding is representable
    x2 = tf32(r1)
    return x1, x2, r1 - x2           # the last 2-3 bits: already a tf32 number


def mm(a, b):
    return (a.astype(f32) @ b.astype(f32)).astype(f32)


def matmul_1xtf32(a, b):
    return mm(tf32(a), tf32(b))


def matmul_3xtf32(a, b):
    ah, al = split2(a)
    bh, bl = split2(b)
    return (mm(al, bh) + mm(ah, bl)) + mm(ah, bh)        # small terms first, as the kernels order their MMAs


def matmul_6x(a, b):
    a1, a2, a3 = split3(a)
    b1, b2, b3 = split3(b)
    small = (mm(a3, b1) + mm(a1, b3)) + mm(a2, b2)
    return (small + (mm(a2, b1) + mm(a1, b2))) + mm(a1, b1)


def matmul_3xtf32_dropped(a, b):
    """3xTF32 with the cross term lo(a) * hi(b) lost: what a projection kernel missing one of its three MMAs computes."""
    ah, _ = split2(a)
    bh, bl = split2(b)
    return mm(ah, bl) + mm(ah, bh)


# Accuracy checks of the split-precision projection rho = X . V (tests/test_projection_gpu.py holds the kernel to them).
#  per element: |rho - X V| <= elementwise_tolerance(D) * (|X| |V|)   -- 2^-20 covers the split (lo*lo dropped, both lo
#               parts rounded to tf32: 3 * 2^-22 per product), D * 2^-23 the float32 accumulation of D products, with a
#               factor 2 for the truncating adds of the tensor cores;
#  normwise:    ||rho - X V||_F / || |X| |V| ||_F  at most normwise_ceiling(D, e) with e that of a float32 FFMA matmul:
#               NORMWISE_FACTOR * sqrt(D / 32) * e.  The tensor cores truncate when they accumulate, so their rounding
#               errors share a sign and grow like D * u where round-to-nearest ones grow like sqrt(D) * u: relative to
#               FFMA the normwise error grows with sqrt(D) (measured on an H100: 2.4x FFMA at D = 32, 6.3x at 256,
#               18x at 2048; this emulation rounds to nearest and stays at ~1x).
# The per-element bound is a ceiling that grows with D, so at D >= ~1024 a lost cross term stays below it; the normwise
# ratio catches that at every D.
NORMWISE_FACTOR = 4.0


def elementwise_tolerance(D):
    return 2.0 ** -20 + D * 2.0 ** -23


def normwise_ceiling(D, ffma_error):
    return NORMWISE_FACTOR * np.sqrt(max(D, 32) / 32.0) * ffma_error


def bound_ratio(got, X, V):
    """max over elements of |got - X V| / (elementwise_tolerance(D) |X| |V|): <= 1 passes."""
    X, V = X.astype(f64), V.astype(f64)
    return float((np.abs(got.astype(f64) - X @ V) / (elementwise_tolerance(X.shape[1]) * (np.abs(X) @ np.abs(V)))).max())


def normwise_error(got, X, V):
    X, V = X.astype(f64), V.astype(f64)
    return float(np.linalg.norm(got.astype(f64) - X @ V) / np.linalg.norm(np.abs(X) @ np.abs(V)))


def test_projection_accuracy_checks_have_teeth():
    """The two checks the wgmma projection must pass: 3xTF32 passes both at every D, plain TF32 and 3xTF32 with one
    cross term lost fail them (the per-element bound alone up to D = 256, the normwise ratio at every D)."""
    rng = np.random.default_rng(4)
    for D in (32, 256, 2048):
        X = rng.standard_normal((2000, D)).astype(f32)
        V = rng.standard_normal((D, 128)).astype(f32)
        ffma = normwise_error(mm(X, V), X, V)
        r3, n3 = bound_ratio(matmul_3xtf32(X, V), X, V), normwise_error(matmul_3xtf32(X, V), X, V)
        assert r3 <= 0.25 and n3 <= normwise_ceiling(D, ffma), (D, r3, n3, ffma)
        for bad in (matmul_1xtf32, matmul_3xtf32_dropped):
            got = bad(X, V)
            rb, nb = bound_ratio(got, X, V), normwise_error(got, X, V)
            assert nb > 5 * normwise_ceiling(D, ffma), (D, bad.__name__, nb, ffma)
            if D <= 256:
                assert rb > 1.0, (D, bad.__name__, rb)


def test_splits_are_exact_where_the_kernels_rely_on_it():
    rng = np.random.default_rng(0)
    x = (rng.standard_normal(100000) * np.exp(rng.uniform(-20, 20, 100000))).astype(f32)
    hi, lo = split2(x)
    assert np.all(np.abs(x.astype(f64) - hi.astype(f64) - lo.astype(f64)) <= 2.0 ** -21 * np.abs(x))   # 22 operand bits
    x1, x2, x3 = split3(x)
    assert np.array_equal(x1.astype(f64) + x2.astype(f64) + x3.astype(f64), x.astype(f64))           # three parts: exact
    for part in (hi, lo, x1, x2, x3):
        assert np.all((part.view(np.uint32) & np.uint32(0x1FFF)) == 0)                                # every part IS a tf32 number


def test_projection_error_plain_vs_split():
    """rho = X . V with D = 256 (VBx/vbhmm.py:129,153 folded into VBx/VBx.py:88-89)."""
    rng = np.random.default_rng(1)
    X = rng.standard_normal((2000, 256))
    V = rng.standard_normal((256, 128)) / 16.0
    ref = X @ V
    scale = np.abs(ref).max()
    e1 = np.abs(matmul_1xtf32(X, V) - ref).max() / scale
    e3 = np.abs(matmul_3xtf32(X, V) - ref).max() / scale
    e6 = np.abs(matmul_6x(X, V) - ref).max() / scale
    ef = np.abs(mm(X, V) - ref).max() / scale
    assert e1 > 1e-4                      # plain TF32: ~3e-4 of the output range, already past the bar before the EM loop
    assert e3 < 5e-6 and e6 < 5e-6        # split: float32-class (measured ~4e-7, same as a float32 matmul)
    assert e3 < 20 * ef and e6 <= e3 * 1.5 + 1e-9


def test_posteriors_need_the_split():
    """One E-step on a synthetic recording (VBx/VBx.py:97 + row softmax) from the reference's default initialisation
    (flat-Dirichlet gamma, VBx/VBx.py:82-83): log-likelihoods from plain TF32 products are off by ~1e-2 and the
    per-frame posteriors by ~5e-4 (bar: 1e-4); from 3xTF32 products by ~3e-5 and ~4e-6.  Later iterations saturate the
    posteriors, but the log-likelihood error - which the ELBO sums over all frames - stays where it is."""
    rng = np.random.default_rng(2)
    T, R, S, Fa, Fb = 1500, 128, 8, 0.3, 17.0
    Phi = synth.plda_phi(R)
    fea, z = synth.make_recording(T, R, Phi, rng, n_spk=5)
    rho = fea * np.sqrt(Phi)[None, :]
    FaFb = Fa / Fb
    for boost in (0.0, 0.05, 1.0):                                   # 0: first iteration; 1.0: posteriors already sharp
        gamma = synth.dirichlet_rows(T, S, np.random.default_rng(3))
        gamma[np.arange(T), z] += boost
        gamma /= gamma.sum(axis=1, keepdims=True)
        invL = 1.0 / (1.0 + FaFb * gamma.sum(axis=0)[:, None] * Phi[None, :])      # VBx/VBx.py:95
        alpha = FaFb * invL * (gamma.T @ rho)                                        # VBx/VBx.py:96
        bias = 0.5 * ((invL + alpha ** 2) * Phi[None, :]).sum(axis=1)

        def e_step(dot):
            ll = Fa * (dot.astype(f64) - bias[None, :])
            p = np.exp(ll - ll.max(axis=1, keepdims=True))
            return ll, p / p.sum(axis=1, keepdims=True)

        ll_ref, post_ref = e_step(rho @ alpha.T)
        ll1, post1 = e_step(matmul_1xtf32(rho, alpha.T))
        ll3, post3 = e_step(matmul_3xtf32(rho, alpha.T))
        assert np.abs(ll1 - ll_ref).max() > 3e-3 and np.abs(ll3 - ll_ref).max() < 1e-4
        assert np.abs(post3 - post_ref).max() < 1e-5
        if boost <= 0.05:
            assert np.abs(post1 - post_ref).max() > 3e-4                # plain TF32: outside the 1e-4 bar
        # the M-step contraction gamma^T . rho (VBx/VBx.py:96) through the same scheme
        ref_m = gamma.T @ rho
        m3 = np.abs(matmul_3xtf32(gamma.T, rho) - ref_m).max() / np.abs(ref_m).max()
        m1 = np.abs(matmul_1xtf32(gamma.T, rho) - ref_m).max() / np.abs(ref_m).max()
        assert m3 < 2e-6 and m1 > 20 * m3
