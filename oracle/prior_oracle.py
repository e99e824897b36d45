"""CPU oracle for the VB-HMM with enrolled speakers as state priors (TEST INFRASTRUCTURE - never on the product path).

A float64 numpy restatement of oracle/vbx_oracle.py's EM loop in which state s's speaker latent starts from the
posterior of y ~ N(0, I) given n_e[s] enrolment x-vectors with feature sum F_e[s] (DESIGN.md section 5.23).  With
c = Fa / Fb the prior is N(mu0, 1/lambda0) per feature,

    lambda0 = 1 + c n_e Phi            mu0 = c sqrt(Phi) F_e / lambda0,

the M-step adds n_e to N_s and sqrt(Phi) F_e to rho^T gamma_s, and the ELBO regulariser is the KL divergence to that
prior instead of to N(0, I).  Everything else is vbx_oracle's.

`augmented_*` state the same model the other way round: the enrolment x-vectors appended to the recording as frames
held on their state (responsibility one-hot, never re-estimated), with the plain N(0, I) prior.  The two views give the
same speaker model, and ELBO_prior = ELBO_augmented - Fb log Z_e, where log Z_e (`log_evidence`) depends on the
enrolment alone.
"""
import math

import numpy as np

from oracle.vbx_oracle import frame_constant, hmm_forward_backward, lse, plda_loglik, speaker_model


def prior_terms(Phi, FaFb, n_e, F_e):
    """lambda0, mu0 [S,R] of the enrolment prior: n_e [S] counts, F_e [S,R] feature sums (fea units)."""
    lam0 = 1.0 + FaFb * np.outer(n_e, Phi)
    mu0 = FaFb * np.sqrt(Phi)[None, :] * F_e / lam0
    return lam0, mu0


def speaker_model_prior(gamma, rho, Phi, FaFb, n_e, F_e):
    """M-step with the enrolment prior.  Returns invL, alpha (S x R)."""
    occupancy = gamma.sum(axis=0) + n_e
    invL = 1.0 / (1.0 + FaFb * np.outer(occupancy, Phi))
    alpha = FaFb * invL * (gamma.T @ rho + np.sqrt(Phi)[None, :] * F_e)
    return invL, alpha


def regulariser_prior(alpha, invL, Phi, Fb, FaFb, n_e, F_e):
    """Fb/2 sum_{s,r} [log(lambda0 invL) - lambda0 invL - lambda0 (alpha - mu0)^2 + 1]: -Fb KL(q || prior)."""
    lam0, mu0 = prior_terms(Phi, FaFb, n_e, F_e)
    d = alpha - mu0
    return 0.5 * Fb * np.sum(np.log(lam0 * invL) - lam0 * invL - lam0 * d * d + 1.0)


def vbx_prior_oracle(X, Phi, prior_n, prior_F, loopProb=0.9, Fa=1.0, Fb=1.0, pi=10, gamma=None, maxIters=10,
                     epsilon=1e-4, return_model=False, alpha=None, invL=None, trace=None):
    """vbx_oracle with the enrolment prior prior_n [S], prior_F [S,R] (zeros: vbx_oracle's results, bit for bit).
    trace: None or a list that receives, per iteration, dict(gamma0, alpha, invL, ll, tll, elbo) (gamma0: the
    responsibilities the iteration started from)."""
    X = np.asarray(X, dtype=np.float64)
    Phi = np.asarray(Phi, dtype=np.float64)
    if type(pi) is int:
        pi = np.full(pi, 1.0 / pi)
    pi = np.asarray(pi, dtype=np.float64)
    S = len(pi)
    n_e = np.asarray(prior_n, dtype=np.float64).reshape(S)
    F_e = np.asarray(prior_F, dtype=np.float64).reshape(S, X.shape[1])
    gamma = np.asarray(gamma, dtype=np.float64)
    G = frame_constant(X)
    rho = X * np.sqrt(Phi)[None, :]
    FaFb = Fa / Fb
    Li = []
    for it in range(maxIters):
        g0 = gamma
        if it > 0 or alpha is None or invL is None:
            invL, alpha = speaker_model_prior(gamma, rho, Phi, FaFb, n_e, F_e)
        ll = plda_loglik(rho, alpha, invL, Phi, G, Fa)
        trans = loopProb * np.eye(S) + (1.0 - loopProb) * pi[None, :]
        gamma, tll, lf, lb = hmm_forward_backward(ll, trans, pi)
        elbo = tll + regulariser_prior(alpha, invL, Phi, Fb, FaFb, n_e, F_e)
        enter = np.exp(lse(lf[:-1], axis=1)[:, None] + ll[1:] + lb[1:] - tll).sum(axis=0)
        pi = gamma[0] + (1.0 - loopProb) * pi * enter
        pi = pi / pi.sum()
        Li.append([float(elbo)])
        if trace is not None:
            trace.append(dict(gamma0=g0, alpha=alpha, invL=invL, ll=ll, tll=tll, elbo=float(elbo)))
        if it > 0 and elbo - Li[-2][0] < epsilon:
            break
    out = (gamma, pi, Li)
    if return_model:
        out = out + (alpha, invL)
    return out


def augmented_model(gamma, X, Phi, FaFb, X_e, state_e):
    """The plain M-step (vbx_oracle.speaker_model) on the recording with the enrolment x-vectors X_e [M,R] appended as
    frames held on their states state_e [M].  Returns invL, alpha."""
    S = gamma.shape[1]
    held = np.zeros((len(X_e), S))
    held[np.arange(len(X_e)), state_e] = 1.0
    rho_a = np.vstack([X, X_e]) * np.sqrt(Phi)[None, :]
    return speaker_model(np.vstack([gamma, held]), rho_a, Phi, FaFb)


def augmented_elbo(tll, alpha, invL, Phi, Fa, Fb, X_e, state_e):
    """The ELBO of the augmented recording: the recording's forward-backward log-likelihood tll, plus the expected
    log-likelihood of every held frame under its state's speaker model, plus the plain regulariser of eq. (25)."""
    rho_e = X_e * np.sqrt(Phi)[None, :]
    held = plda_loglik(rho_e, alpha, invL, Phi, frame_constant(X_e), Fa)[np.arange(len(X_e)), state_e]
    return tll + held.sum() + 0.5 * Fb * np.sum(np.log(invL) - invL - alpha * alpha + 1.0)


def log_evidence(Phi, Fa, Fb, X_e, state_e, S):
    """log Z_e = sum_s log integral N(y; 0, I) prod_{e on s} p(x_e | y)^(Fa/Fb) dy of the PLDA model of VBx (x | y ~
    N(sqrt(Phi) y, I)), in closed form per feature: the constant between the two ELBOs is Fb log Z_e."""
    c = Fa / Fb
    out = 0.0
    for s in range(S):
        x = X_e[state_e == s]
        n = len(x)
        if n == 0:
            continue
        lam0 = 1.0 + c * n * Phi
        b = c * np.sqrt(Phi) * x.sum(axis=0)
        quad = -0.5 * c * np.sum(x * x) - 0.5 * c * n * len(Phi) * math.log(2.0 * math.pi)
        out += quad + np.sum(0.5 * b * b / lam0 - 0.5 * np.log(lam0))
    return float(out)
