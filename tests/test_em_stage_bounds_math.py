"""The accuracy checks tests/test_em_stages_gpu.py holds the in-loop kernels to, restated in numpy and shown to have teeth:
the split-precision 3xTF32 contractions (emulated bit-level as in tests/test_split_precision_math.py) pass them, plain TF32
and 3xTF32 with one cross term lost fail them, at the shapes the GPU tests use.

Stage 1, M-step + speaker model (VBx/VBx.py:95-96), per recording:
    Sigma[s,r] = sum_t gamma[t,s] rho[t,r]   float32 tile sums over <= kMTile = 512 frames, float64 across tiles
    invL       = 1 / (1 + FaFb N_s Phi_r)    float32, N_s the float32 rounding of a float64 sum
    alpha      = float32(float64(float32(FaFb invL)) Sigma)
  Per element, with u = 2^-24 and c = FaFb invL (float64):
    |invL - invL_ref|   <= INVL_ULPS u invL_ref                 N_s, FaFb, the product, the add and the divide: <= 6 u
    |alpha - alpha_ref| <= c elementwise_tolerance(512) sum_t gamma |rho|   the tile sums (one tile's bound covers the
                                                                           float64 sum of several)
                           + ALPHA_ULPS u |alpha_ref|           c carries invL's 8 u, FaFb's and the product's u, then
                                                                the final rounding: 11 u, rounded up to 12
  Normwise, Sigma backed out as alpha / c:  ||Sigma - Sigma_ref||_F / || gamma^T |rho| ||_F  at most
    MSTEP_NORMWISE_FACTOR normwise_ceiling(512, e) + ALPHA_ULPS u, e the same ratio of a float32 FFMA of the same tiles.
    MSTEP_NORMWISE_FACTOR = 3: at S >= 64 one warp accumulates all 512 frames of a tile in the tensor cores' truncating
    adds, a longer chain than the projection's (measured on an H100 at 700 W: 1.46 times normwise_ceiling at S = 128).
Stage 2, log-likelihood (VBx/VBx.py:97) from a given float32 model, per frame t and state s:
    ll[t,s] = rho_t . A_s - bias_s,  A = float32(Fa alpha) split hi/lo,  bias_s = Fa/2 sum_r (invL + alpha^2) Phi_r
    E[t,s]  = elementwise_tolerance(R) sum_r |rho_tr| |A_sr|   the contraction of R products
              + 3 u sum_r |rho_tr| |A_sr|                    rho = fea sqrt(Phi) and A = Fa alpha rounded to float32
              + BIAS_ULPS u |bias_s| + 2 u |ll[t,s]|         bias: float32 groups of 32 terms; ll itself stored in float32
  The kernels' ll is seen through gamma: with loopProb = 0 a gamma row is the normalised p_t w, so
  log gamma[t,s] - log w_s equals ll[t,s] up to a per-frame constant.  Centred over the live states of the frame, the
  device's and the float64 ll differ per element by at most  E[t,s] + mean_j E[t,j] + 2 GAMMA_ULPS u  (the rounding of
  the two gamma values, relative GAMMA_ULPS u each), and normwise by at most normwise_ceiling(R, e) plus the same
  rounding term, e the centred float32 FFMA error over || sum_r |rho| |A| ||_F.
"""
import numpy as np

from test_split_precision_math import (elementwise_tolerance, matmul_1xtf32, matmul_3xtf32, matmul_3xtf32_dropped, mm,
                                       normwise_ceiling)

f32, f64 = np.float32, np.float64
U = 2.0 ** -24
K_MTILE = 512
INVL_ULPS = 8
ALPHA_ULPS = 12
BIAS_ULPS = 48
GAMMA_ULPS = 64
MSTEP_NORMWISE_FACTOR = 3.0


def tile_sums(gamma, rho, matmul):
    """Sigma = gamma^T rho of one recording: `matmul` in float32 over each 512-frame tile, float64 across tiles."""
    S, R = gamma.shape[1], rho.shape[1]
    out = np.zeros((S, R))
    for t0 in range(0, gamma.shape[0], K_MTILE):
        out += matmul(gamma[t0:t0 + K_MTILE].T, rho[t0:t0 + K_MTILE]).astype(f64)
    return out


def speaker_model_ref(gamma, rho, Phi, Fa, Fb):
    """float64 (N_s, Sigma, invL, alpha) of one recording from the float32 gamma and rho the device holds."""
    g, x = gamma.astype(f64), rho.astype(f64)
    Ns = g.sum(0)
    Sig = g.T @ x
    invL = 1.0 / (1.0 + (Fa / Fb) * Ns[:, None] * Phi.astype(f64)[None, :])
    return Ns, Sig, invL, (Fa / Fb) * invL * Sig


def speaker_model_f32(Sig, Ns, Phi, Fa, Fb):
    """invL and alpha as speaker_model_kernel computes them from the tile sums Sigma (float64)."""
    FaFb = f32(Fa / Fb)
    invL = (f32(1) / (f32(1) + FaFb * Ns.astype(f32)[:, None] * Phi.astype(f32)[None, :])).astype(f32)
    alpha = ((FaFb * invL).astype(f32).astype(f64) * Sig).astype(f32)
    return invL, alpha


def alpha_bound(gamma, rho, Phi, Fa, Fb):
    """Per-element bound on |alpha - alpha_ref| (module docstring) and alpha_ref."""
    _, _, invL, alpha = speaker_model_ref(gamma, rho, Phi, Fa, Fb)
    c = (Fa / Fb) * invL
    gabs = gamma.astype(f64).T @ np.abs(rho.astype(f64))
    return c * elementwise_tolerance(K_MTILE) * gabs + ALPHA_ULPS * U * np.abs(alpha), alpha


def mstep_errors(recs, Phi, Fa, Fb, alphas, invLs):
    """Worst per-element ratios of invL and alpha to their bounds and the normwise error of Sigma over recordings `recs`
    [(gamma, rho)] with the device's (alpha, invL) per recording.  Returns (invL ratio, alpha ratio, normwise, ceiling)."""
    r_inv = r_alpha = 0.0
    num = den = num_f = 0.0
    for (g, x), a, il in zip(recs, alphas, invLs):
        if g.shape[0] == 0:
            continue
        bound, a_ref = alpha_bound(g, x, Phi, Fa, Fb)
        Ns, Sig, il_ref, _ = speaker_model_ref(g, x, Phi, Fa, Fb)
        r_inv = max(r_inv, float((np.abs(il.astype(f64) - il_ref) / (INVL_ULPS * U * il_ref)).max()))
        r_alpha = max(r_alpha, float((np.abs(a.astype(f64) - a_ref) / bound).max()))
        c_dev = (f32(Fa / Fb) * il.astype(f32)).astype(f32).astype(f64)
        sig_dev = a.astype(f64) / c_dev
        gabs = g.astype(f64).T @ np.abs(x.astype(f64))
        num += float(((sig_dev - Sig) ** 2).sum())
        den += float((gabs ** 2).sum())
        num_f += float(((tile_sums(g, x, mm) - Sig) ** 2).sum())
    nw, e_ffma = np.sqrt(num / den), np.sqrt(num_f / den)
    return r_inv, r_alpha, nw, MSTEP_NORMWISE_FACTOR * normwise_ceiling(K_MTILE, e_ffma) + ALPHA_ULPS * U


def loglik_parts(rho, alpha, invL, Phi, Fa):
    """float64 ll [T,S], the per-element bound E [T,S] and the magnitudes sum_r |rho| |A| of one recording from the float32
    model the device was given."""
    x = rho.astype(f64)
    A = Fa * alpha.astype(f64)
    bias = 0.5 * Fa * ((invL.astype(f64) + alpha.astype(f64) ** 2) * Phi.astype(f64)[None, :]).sum(1)
    ll = x @ A.T - bias[None, :]
    mag = np.abs(x) @ np.abs(A).T
    R = rho.shape[1]
    E = (elementwise_tolerance(R) + 3 * U) * mag + BIAS_ULPS * U * np.abs(bias)[None, :] + 2 * U * np.abs(ll)
    return ll, E, mag


def centred(v, live):
    """v [T,S] minus its per-frame mean over the entries where live [T,S] holds; 0 elsewhere."""
    n = np.maximum(live.sum(1, keepdims=True), 1)
    m = np.where(live, v, 0.0).sum(1, keepdims=True) / n
    return np.where(live, v - m, 0.0)


def loglik_errors(recs, Phi, Fa, gammas, ws, gamma_refs, ffma_ll):
    """recs [(rho, alpha, invL)] per recording, gammas the device's gamma (live columns), ws the transition weights w,
    gamma_refs the float64 gamma, ffma_ll the float32 FFMA ll per recording (the normwise yardstick).  Returns (worst
    per-element ratio, normwise error, ceiling)."""
    worst = 0.0
    num = den = num_f = cnt = 0.0
    for (x, a, il), g, w, gr, lf in zip(recs, gammas, ws, gamma_refs, ffma_ll):
        if x.shape[0] == 0:
            continue
        ll, E, mag = loglik_parts(x, a, il, Phi, Fa)
        live = (gr > 1e-20) & (g.astype(f64) > 1e-20)
        with np.errstate(divide='ignore'):
            lw = np.log(w)[None, :]
            d_dev = centred(np.log(np.where(live, g.astype(f64), 1.0)) - lw, live)
        d_ref = centred(ll, live)
        err = np.abs(d_dev - d_ref)
        n = np.maximum(live.sum(1, keepdims=True), 1)
        bound = E + np.where(live, E, 0.0).sum(1, keepdims=True) / n + 2 * GAMMA_ULPS * U
        worst = max(worst, float(np.where(live, err / bound, 0.0).max()))
        num += float((err[live] ** 2).sum())
        den += float((mag[live] ** 2).sum())
        num_f += float(((centred(lf.astype(f64), live) - d_ref)[live] ** 2).sum())
        cnt += float(live.sum())
    nw = np.sqrt(num / den)
    return worst, nw, normwise_ceiling(recs[0][0].shape[1], np.sqrt(num_f / den)) + 2 * GAMMA_ULPS * U * np.sqrt(cnt / den)


def ll_emulated(rho, alpha, invL, Phi, Fa, matmul):
    """ll as the log-likelihood kernels compute it: rho . float32(Fa alpha) through `matmul`, minus bias (float32)."""
    A = (f32(Fa) * alpha.astype(f32)).astype(f32)
    bias = (0.5 * Fa * ((invL.astype(f64) + alpha.astype(f64) ** 2) * Phi.astype(f64)[None, :]).sum(1)).astype(f32)
    return (matmul(rho.astype(f32), A.T) - bias[None, :]).astype(f32)


def posterior(ll, w):
    """gamma of a loopProb = 0 sweep: p_t w normalised per frame, float64."""
    z = ll.astype(f64) + np.log(w)[None, :]
    z -= z.max(1, keepdims=True)
    e = np.exp(z)
    return e / e.sum(1, keepdims=True)


def synthetic(T, R, S, seed, offset=0.0):
    rng = np.random.default_rng(seed)
    Phi = np.exp(np.linspace(np.log(5.6), np.log(0.53), R)).astype(f32)
    rho = ((rng.standard_normal((T, R)) + offset) * np.sqrt(Phi)[None, :]).astype(f32)
    g = rng.gamma(1.0, size=(T, S))
    return Phi, rho, (g / g.sum(1, keepdims=True)).astype(f32)


def test_mstep_bounds_have_teeth():
    """3xTF32 tile sums pass the stage-1 bounds at every feature width the GPU tests run; plain TF32 and either lost
    cross term (gamma's or rho's low part) break the normwise ceiling by more than twice."""
    Fa, Fb = 0.3, 17.0
    for R, S, T in ((4, 4, 1100), (12, 16, 700), (52, 16, 1025), (128, 64, 1500)):
        Phi, rho, g = synthetic(T, R, S, seed=R + S)
        errs = {}
        for name, matmul in (('3x', matmul_3xtf32), ('1x', matmul_1xtf32), ('drop_lo_gamma', matmul_3xtf32_dropped),
                             ('drop_lo_rho', lambda a, b: matmul_3xtf32_dropped(b.T, a.T).T)):
            Ns = g.astype(f64).sum(0)
            invL, alpha = speaker_model_f32(tile_sums(g, rho, matmul), Ns, Phi, Fa, Fb)
            errs[name] = mstep_errors([(g, rho)], Phi, Fa, Fb, [alpha], [invL])
        r_inv, r_a, nw, ceil = errs['3x']
        print(f'R={R} S={S} T={T}: 3xTF32 invL {r_inv:.3g} alpha {r_a:.3g} normwise {nw / ceil:.3g} of the ceiling; '
              + ' '.join(f'{k} {v[2] / v[3]:.3g}' for k, v in errs.items() if k != '3x'))
        assert r_inv <= 1 and r_a <= 1 and nw <= ceil, (R, errs['3x'])
        for bad in ('1x', 'drop_lo_gamma', 'drop_lo_rho'):
            assert errs[bad][2] > 2 * errs[bad][3], (R, bad, errs[bad])


def test_loglik_bounds_have_teeth():
    """The stage-2 checks through gamma: 3xTF32 passes them at every width, plain TF32 and a lost cross term break the
    normwise ceiling (and, at R = 128, the per-element bound)."""
    Fa = 0.3
    for R, S, T in ((4, 4, 600), (12, 16, 600), (52, 16, 600), (100, 64, 400), (128, 16, 1200)):
        Phi, rho, _ = synthetic(T, R, S, seed=3 * R + S)
        rng = np.random.default_rng(R)
        alpha = (0.6 * rng.standard_normal((S, R)) * np.sqrt(Phi)[None, :]).astype(f32)
        invL = rng.uniform(0.02, 0.6, (S, R)).astype(f32)
        w = rng.dirichlet(np.ones(S)) + 1e-8
        ll_ref, _, _ = loglik_parts(rho, alpha, invL, Phi, Fa)
        g_ref = posterior(ll_ref, w)
        ffma = ll_emulated(rho, alpha, invL, Phi, Fa, mm)
        res = {}
        for name, matmul in (('3x', matmul_3xtf32), ('1x', matmul_1xtf32), ('drop', matmul_3xtf32_dropped)):
            g = posterior(ll_emulated(rho, alpha, invL, Phi, Fa, matmul), w).astype(f32)
            res[name] = loglik_errors([(rho, alpha, invL)], Phi, Fa, [g], [w], [g_ref], [ffma])
        print(f'R={R} S={S}: ' + ' '.join(f'{k} elem {v[0]:.3g} normwise {v[1] / v[2]:.3g}' for k, v in res.items()))
        assert res['3x'][0] <= 1 and res['3x'][1] <= res['3x'][2], (R, res['3x'])
        for bad in ('1x', 'drop'):
            assert res[bad][1] > 3 * res[bad][2], (R, bad, res[bad])
        if R == 128:
            assert res['1x'][0] > 1, res['1x']
