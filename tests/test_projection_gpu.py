"""The tensor-core front end (vbx_project_tc.cu) against float64 at every tile edge: the wgmma projection rho = X . V
(MODE 0), the x-vector chain (MODE 1 -> MODE 2), the per-frame ELBO constant G_t of every prepare path, and batches
holding recordings without frames.

Frame counts NS_EDGE cover a partial single tile, one tile per CTA of the persistent grid (one CTA per SM), some CTAs
with one tile more than the others, and 1, 2 or 3 tiles per CTA; with D / 32 pipeline blocks per tile that gives odd and
even block counts per producer.  Where the arithmetic allows it the result is checked bit for bit: the exact probes
make every output element a single product whose operands are exactly hi + lo (or x1 + x2 + x3) of the split, so any
layout, swizzle, stage, tail-row or missing-term error changes bits."""
import math
import os

import numpy as np
import pytest
import torch

from test_split_precision_math import elementwise_tolerance, normwise_ceiling, split2
from vbx_b200 import pipeline, synth

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), 'golden')
DS = [32, 64, 96, 128, 160, 256, 512, 2048]
LOG2PI = math.log(2.0 * math.pi)


def dev():
    return torch.device('cuda:0')


def cuda(a, dtype=torch.float32):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev()).to(dtype)


def ns_edge():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return sorted({1, 63, 64, 65, 127, 128, 129, 128 * sms - 1, 128 * sms, 128 * sms + 1, 128 * (2 * sms + 1) + 5})


def new_batch(lengths, S=4, **kw):
    from vbx_b200.batch import VbxBatch
    vb = VbxBatch(lengths, 128, S, device=dev(), **kw)
    vb.workspace.fill_(0xFF)          # NaN in float32 and float64: nothing may be read before it is written
    return vb


GUARD = 128


def project(vb, X, V, Phi, path):
    """rho through one projection path (1 = FFMA, 2 = wgmma), written into a buffer followed by NaN guard rows: a store
    to a frame >= N shows up there."""
    N = X.shape[0]
    vb.set_option('projection', path)
    buf = torch.full((N + GUARD, 128), float('nan'), device=dev())
    rho = vb.prepare_project(X, V, Phi, out=buf[:N])
    torch.cuda.synchronize()
    assert torch.isnan(buf[N:]).all(), 'projection stored past the last frame'
    return rho


def assert_bits_equal(got, want, what):
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()
    t, n = (int(v) for v in bad[0])
    raise AssertionError(f'{what}: {bad.shape[0]} elements differ, first at frame {t} (tile {t // 128}, row {t % 128}) '
                         f'column {n}: got {float(got[t, n])!r}, want {float(want[t, n])!r}')


def bits22_pool(rng, n=4096):
    """Values with exactly 22 significant bits (odd 22-bit mantissas): x == hi + lo exactly under the two-way split
    and lo != 0, so a product of two of them, or of one and a power of two, is what 3xTF32 computes without rounding."""
    m = rng.integers(2 ** 21, 2 ** 22, n) | 1
    x = (rng.choice([-1.0, 1.0], n) * m * 2.0 ** (rng.integers(-4, 5, n) - 21)).astype(np.float32)
    hi, lo = split2(x)
    assert np.array_equal(hi.astype(np.float64) + lo.astype(np.float64), x.astype(np.float64))
    assert np.all(lo != 0)
    return cuda(x)


# ---------------------------------------------------------------- a. exact layout probes (MODE 0) --------------------

@pytest.mark.parametrize('D', DS)
def test_projection_probe_selection(D):
    """V is a 0/1 selection matrix (one 1 per output column): rho == X[:, sel] bit for bit, over enough launches that
    every input column is selected (the first and last column of every 32-wide block included)."""
    rng = np.random.default_rng(D)
    pool = bits22_pool(rng)
    perm = rng.permutation(D)
    cols = np.resize(perm, -(-D // 128) * 128)
    Phi = torch.ones(128, device=dev())
    for N in ns_edge():
        g = torch.Generator(device=dev()).manual_seed(N)
        X = pool[torch.randint(0, pool.numel(), (N, D), generator=g, device=dev())]
        vb = new_batch([N])
        for j in range(cols.size // 128):
            sel = cols[128 * j:128 * (j + 1)]
            V = torch.zeros((D, 128), device=dev())
            V[torch.from_numpy(sel).to(dev()), torch.arange(128, device=dev())] = 1.0
            rho = project(vb, X, V, Phi, 2)
            assert_bits_equal(rho, X[:, torch.from_numpy(sel).to(dev())], f'D={D} N={N} launch {j}')
        vb.close()


@pytest.mark.parametrize('D', DS)
def test_projection_probe_one_hot_rows(D):
    """Rows of X are one-hot, the hot column k(t) moving with the row inside the tile and with the tile:
    rho[t] == V[k(t)] bit for bit."""
    rng = np.random.default_rng(100 + D)
    pool = bits22_pool(rng)
    Phi = torch.ones(128, device=dev())
    g = torch.Generator(device=dev()).manual_seed(D)
    V = pool[torch.randint(0, pool.numel(), (D, 128), generator=g, device=dev())]
    for N in ns_edge():
        t = torch.arange(N, device=dev())
        k = ((t % 128) * 37 + (t // 128) * 11 + N) % D
        X = torch.zeros((N, D), device=dev())
        X[t, k] = 1.0
        vb = new_batch([N])
        rho = project(vb, X, V, Phi, 2)
        assert_bits_equal(rho, V[k], f'D={D} N={N}')
        vb.close()


# ---------------------------------------------------------------- b. accuracy, per element and normwise --------------

def projection_inputs(kind, N, D, gen):
    """X [N,D], V [D,128] float32 on the device.  'cancel': rows of X carry a large common offset that the columns of V
    are (nearly) orthogonal to, so |x . v| << |x| . |v|, as with the shipped LDA on raw x-vectors."""
    X = torch.randn((N, D), generator=gen, device=dev())
    if kind == 'random':
        V = torch.randn((D, 128), generator=gen, device=dev())
    elif kind == 'basis':
        B = synth.projection_basis(D, 128) if D >= 128 else synth.projection_basis(128, D).T
        V = cuda(B * np.sqrt(synth.plda_phi(128))[None, :])
    else:
        mu = torch.randn(D, generator=gen, device=dev(), dtype=torch.float64)
        mu /= mu.norm()
        W = torch.randn((D, 128), generator=gen, device=dev(), dtype=torch.float64)
        V = (W - mu[:, None] * (mu @ W)[None, :]).float()
        X = X + 100.0 * mu.float()[None, :]
    return X.contiguous(), V.contiguous()


def projection_errors(rho, X, V, chunk=1 << 19):
    """(max over elements of |rho - X V| / (elementwise_tolerance(D) |X||V|), normwise error); float64 on the device,
    every element, in row chunks."""
    V64 = V.double()
    tol = elementwise_tolerance(X.shape[1])
    worst, e2, m2 = 0.0, 0.0, 0.0
    for i in range(0, X.shape[0], chunk):
        x = X[i:i + chunk].double()
        err = (rho[i:i + chunk].double() - x @ V64).abs()
        mag = x.abs() @ V64.abs()
        worst = max(worst, float((err / (tol * mag)).max()))
        e2 += float((err ** 2).sum())
        m2 += float((mag ** 2).sum())
    return worst, math.sqrt(e2 / m2)


@pytest.mark.parametrize('kind', ['random', 'basis', 'cancel'])
@pytest.mark.parametrize('D', DS)
def test_projection_accuracy_bounds(D, kind):
    """Every element within the split + accumulation bound, and the normwise error within normwise_ceiling of the FFMA
    path on the same inputs (tests/test_split_precision_math.py derives both and shows that a lost term fails them)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    gen = torch.Generator(device=dev()).manual_seed(7 * D + len(kind))
    Phi = cuda(synth.plda_phi(128))
    for N in (1, 129, 128 * (2 * sms + 1) + 5):
        X, V = projection_inputs(kind, N, D, gen)
        vb = new_batch([N])
        worst, nw = projection_errors(project(vb, X, V, Phi, 2), X, V)
        _, nf = projection_errors(project(vb, X, V, Phi, 1), X, V)
        vb.close()
        print(f'D={D} {kind} N={N}: max err / bound {worst:.3g}, normwise wgmma {nw:.3g} FFMA {nf:.3g}')
        assert worst <= 1.0, (D, kind, N, worst)
        if N > 128:            # a handful of elements says nothing about the typical error
            assert nw <= normwise_ceiling(D, nf), (D, kind, N, nw, nf)


def test_projection_accuracy_at_the_benchmark_shape():
    """The benchmark's headline shape, N = 4096 x 1000 frames, D = 256 (about 242 tiles per CTA on 132 SMs): every
    element of rho against a float64 matmul on the device."""
    N, D = 4096 * 1000, 256
    gen = torch.Generator(device=dev()).manual_seed(2024)
    X = torch.randn((N, D), generator=gen, device=dev())
    V = cuda(synth.projection_basis(D, 128) * np.sqrt(synth.plda_phi(128))[None, :])
    Phi = cuda(synth.plda_phi(128))
    vb = new_batch([1000] * 4096)
    worst, nw = projection_errors(project(vb, X, V, Phi, 2), X, V)
    _, nf = projection_errors(project(vb, X, V, Phi, 1), X, V)
    vb.close()
    print(f'headline shape: max err / bound {worst:.3g}, normwise wgmma {nw:.3g} FFMA {nf:.3g}')
    assert worst <= 1.0, worst
    assert nw <= normwise_ceiling(D, nf), (nw, nf)


# ---------------------------------------------------------------- c. the x-vector chain (MODE 1 -> MODE 2) -----------

def xvector_model(rng, Dx):
    """The shapes of the shipped model (Dx -> LDA 128 -> PLDA 128); LDA columns scaled so that |x_lda| ~ 1 and the
    subtracted mean2 is a sizeable part of it."""
    mean1 = rng.standard_normal(Dx) * 0.5
    lda = rng.standard_normal((Dx, 128)) / np.sqrt(128)
    mean2 = rng.standard_normal(128) * 0.05
    plda_mu = rng.standard_normal(128) * 0.02
    q, _ = np.linalg.qr(rng.standard_normal((128, 128)))
    plda_tr = q * rng.uniform(2.0, 20.0, 128)[:, None]
    plda_psi = np.exp(rng.uniform(-2.0, 2.0, 128))
    return [np.ascontiguousarray(a, dtype=np.float32) for a in (mean1, lda, mean2, plda_mu, plda_tr, plda_psi)]


def chain_reference(x_raw, model):
    """The float64 host chain (vbx_b200.pipeline) on the float32 inputs, on the device: (x_norm, rho)."""
    mean1, lda, mean2, mu, tr, psi = (cuda(a, torch.float64) for a in model)
    xn = pipeline.xvector_transform(x_raw.double(), mean1, mean2, lda)
    return xn, pipeline.plda_project(xn, mu, tr, 128) * psi.sqrt()[None, :]


def run_chain(x_raw, model):
    vb = new_batch([x_raw.shape[0]])
    rho, x_norm = vb.prepare_xvectors(x_raw, *(cuda(a) for a in model))
    torch.cuda.synchronize()
    vb.close()
    return rho, x_norm


@pytest.mark.parametrize('Dx', [32, 64, 256, 512, 2048])
def test_xvector_chain_per_row(Dx):
    """Both passes against the float64 chain row by row: every x_norm row against its reference unit vector, every rho
    row relative to its own size, |x_norm_t| = 1.  Row scales spread over e^+-2, so a row norm taken from another row
    or another tile (the MODE 1 norm buffer alternates with the tile parity) changes x_norm far beyond the bound.
    The bounds are those of test_parity_gpu.py at Dx = 256, grown in proportion to Dx above it: the truncating
    tensor-core accumulation gives a relative error ~ sqrt(Dx) * u of sum |x_k lda_kn|, itself ~ sqrt(Dx) x |x . lda|
    (measured on an H100: x_norm 6.4e-7, 1.3e-6, 4.2e-6 at Dx = 256, 512, 2048)."""
    rng = np.random.default_rng(300 + Dx)
    model = xvector_model(rng, Dx)
    grow = max(Dx, 256) / 256
    for N in ns_edge():
        scale = np.exp(rng.uniform(-2.0, 2.0, (N, 1)))
        x_raw = cuda(model[0][None, :] + rng.standard_normal((N, Dx)) * scale)
        rho, x_norm = run_chain(x_raw, model)
        xn64, rho64 = chain_reference(x_raw, model)
        ex = (x_norm.double() - xn64).abs().amax(1)
        er = (rho.double() - rho64).abs().amax(1) / rho64.abs().amax(1)
        en = (x_norm.double().norm(dim=1) - 1.0).abs()
        print(f'Dx={Dx} N={N}: x_norm {float(ex.max()):.2e}, rho {float(er.max()):.2e}, |x_norm|-1 {float(en.max()):.2e}')
        assert float(ex.max()) <= 4e-6 * grow, (Dx, N, int(ex.argmax()), float(ex.max()))
        assert float(er.max()) <= 1e-5 * grow, (Dx, N, int(er.argmax()), float(er.max()))
        assert float(en.max()) <= 1e-6, (Dx, N, int(en.argmax()), float(en.max()))


def test_xvector_chain_second_pass_exact():
    """plda_tr a signed permutation and plda_psi powers of 4 (sqrt and 1/psi exact): the PLDA pass is one exact
    product per element, rho == fp32(x_norm - plda_mu)[:, perm] * sign * 2^k bit for bit, with x_norm as returned."""
    rng = np.random.default_rng(11)
    model = xvector_model(rng, 256)
    perm = rng.permutation(128)
    sign = rng.choice([-1.0, 1.0], 128)
    k = rng.integers(-3, 4, 128)
    tr = np.zeros((128, 128))
    tr[np.arange(128), perm] = sign
    model[4] = tr.astype(np.float32)
    model[5] = (4.0 ** k).astype(np.float32)
    mu = cuda(model[3])
    scale = cuda(sign * 2.0 ** k)
    for N in ns_edge():
        x_raw = cuda(model[0][None, :] + rng.standard_normal((N, 256)) * 2.0)
        rho, x_norm = run_chain(x_raw, model)
        want = (x_norm - mu[None, :])[:, torch.from_numpy(perm).to(dev())] * scale[None, :]
        assert_bits_equal(rho, want, f'N={N}')


def test_xvector_chain_shipped_model():
    """The shipped model (its LDA is badly conditioned) on seeded random x-vectors with the spread of the ES2005a ones,
    at the tolerances of test_pipeline.py::test_es2005a_raw_xvectors_to_rttm_on_gpu."""
    m = np.load(os.path.join(GOLD, 'es2005a_model.npz'))
    es = np.load(os.path.join(GOLD, 'es2005a.npz'))
    model = [np.ascontiguousarray(m[k], dtype=np.float32) for k in ('mean1', 'lda', 'mean2', 'plda_mu', 'plda_tr', 'plda_psi')]
    mean, std = es['x_raw'].mean(0), es['x_raw'].std(0)
    rng = np.random.default_rng(21)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for N in (1, 129, 128 * sms + 1, 128 * (2 * sms + 1) + 5):
        x_raw = cuda(mean[None, :] + rng.standard_normal((N, mean.size)) * std[None, :])
        rho, x_norm = run_chain(x_raw, model)
        xn64, rho64 = chain_reference(x_raw, model)
        sq = cuda(model[5], torch.float64).sqrt()[None, :]
        e_x = float((x_norm.double() - xn64).abs().max())
        e_f = float(((rho.double() - rho64) / sq).abs().max())
        print(f'shipped model N={N}: max |x_norm - ref| {e_x:.2e}, max |fea - ref| {e_f:.2e}')
        assert e_x <= 1.5e-5 and e_f <= 3e-4, (N, e_x, e_f)


# ---------------------------------------------------------------- d. the ELBO constant of every prepare path ---------

LENS_RAGGED = [0, 1, 127, 128, 0, 129, 511, 512, 513, 4500, 0]


def g_reference(rho, Phi, lengths):
    """-0.5 sum_t (sum_r rho_tr^2 / Phi_r + R log 2pi) per recording, float64, from the returned rho."""
    q = (rho.double() ** 2 / Phi.double()[None, :]).sum(1) + 128 * LOG2PI
    cs = torch.cat([torch.zeros(1, dtype=torch.float64, device=dev()), torch.cumsum(q, 0)])
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(lengths)])).to(dev())
    return -0.5 * (cs[off[1:]] - cs[off[:-1]])


def check_g(got, want, lengths, what, rtol=1e-6):
    got, want = got.cpu().numpy(), want.cpu().numpy()
    empty = np.asarray(lengths) == 0
    assert np.all(got[empty] == 0.0), (what, got[empty])
    rel = np.abs(got - want)[~empty] / np.abs(want[~empty])
    assert rel.max() <= rtol, (what, int(np.flatnonzero(~empty)[rel.argmax()]), rel.max())


@pytest.mark.parametrize('lengths', [LENS_RAGGED, [1] * 300], ids=['ragged', 'single_frames'])
def test_g_sum_of_every_prepare_path(lengths):
    """g_sum() after prepare_scale, prepare_project (wgmma and FFMA) and prepare_xvectors against float64 from the
    returned rho.  With one-frame recordings every entry is a single G_t, so a G_t stored for the wrong frame shows;
    Phi has distinct entries, so a wrong 1/Phi column shows."""
    rng = np.random.default_rng(len(lengths))
    N = int(sum(lengths))
    Phi = cuda(np.exp(rng.uniform(-2.0, 2.0, 128)))
    vb = new_batch(lengths)
    fea = cuda(rng.standard_normal((N, 128)))
    rho = vb.prepare_scale(fea, Phi)
    check_g(vb.g_sum(), g_reference(rho, Phi, lengths), lengths, 'prepare_scale')
    X = cuda(rng.standard_normal((N, 256)))
    V = cuda(synth.projection_basis(256, 128) * np.sqrt(Phi.double().cpu().numpy())[None, :])
    gs = {}
    for path in (2, 1):
        vb.workspace.fill_(0xFF)
        rho = project(vb, X, V, Phi, path)
        gs[path] = vb.g_sum()
        check_g(gs[path], g_reference(rho, Phi, lengths), lengths, f'prepare_project path {path}')
    # Across the two GEMMs G also carries their difference: the truncating tensor-core adds shrink |rho| by ~1e-6
    # relative at D = 256 (measured on an H100: wgmma and FFMA G differ by 0.9e-6 ... 1.5e-6), and G is quadratic in rho.
    check_g(gs[2], gs[1], lengths, 'wgmma against FFMA', rtol=4e-6)
    model = xvector_model(rng, 256)
    vb.workspace.fill_(0xFF)
    x_raw = cuda(model[0][None, :] + rng.standard_normal((N, 256)))
    rho, _ = vb.prepare_xvectors(x_raw, *(cuda(a) for a in model))
    check_g(vb.g_sum(), g_reference(rho, cuda(model[5]), lengths), lengths, 'prepare_xvectors')
    vb.close()


def test_g_sum_of_a_batch_without_frames():
    """Recordings without frames only: every prepare path still writes G = 0 for each of them."""
    lengths = [0, 0, 0]
    vb = new_batch(lengths)
    Phi = torch.ones(128, device=dev())
    empty = lambda D: torch.zeros((0, D), device=dev())
    vb.prepare_scale(empty(128), Phi)
    assert torch.equal(vb.g_sum(), torch.zeros(3, dtype=torch.float64, device=dev()))
    for path in (2, 1):
        vb.workspace.fill_(0xFF)
        vb.set_option('projection', path)
        vb.prepare_project(empty(256), torch.zeros((256, 128), device=dev()), Phi)
        assert torch.equal(vb.g_sum(), torch.zeros(3, dtype=torch.float64, device=dev())), path
    vb.workspace.fill_(0xFF)
    model = [cuda(a) for a in xvector_model(np.random.default_rng(0), 64)]
    vb.prepare_xvectors(empty(64), *model)
    assert torch.equal(vb.g_sum(), torch.zeros(3, dtype=torch.float64, device=dev()))
    vb.close()


def test_g_sum_needs_a_prepare_call():
    from vbx_b200 import VbxError
    vb = new_batch([5, 7])
    with pytest.raises(VbxError):
        vb.g_sum()
    vb.close()


# ---------------------------------------------------------------- e. recordings without frames inside a batch -------

@pytest.mark.parametrize('fb', [2, 1], ids=['fused', 'split'])
def test_empty_recordings_in_a_batch(fb):
    """T = 0 recordings first, in the middle and last: they run no iteration (n_iters 0, flags 0, Li all NaN, G 0,
    their pi row untouched), and every other recording's results are bit-identical to the batch without them.  A finite
    epsilon, so the float64 finishing phase runs too."""
    lens = [300, 45, 129, 600]
    with_empty = [0, 300, 45, 0, 129, 600, 0]
    S = 8
    d = synth.make_batch(lens, R=128, S=S, seed=31, D=256, dtype=np.float32)
    kw = dict(Fa=0.3, Fb=17.0, loopProb=0.99, maxIters=30, epsilon=1e-5)

    def run(lengths):
        vb = new_batch(lengths, S=S, fb_split=fb)
        vb.prepare_project(cuda(d['X']), cuda(d['V']), cuda(d['Phi']))
        g = cuda(d['gamma0'])
        p = torch.full((len(lengths), S), 1.0 / S, device=dev())
        out = vb.run(g, p, return_model=True, **kw)
        G = vb.g_sum()
        torch.cuda.synchronize()
        res = {k: out[k].cpu().numpy() for k in ('gamma', 'pi', 'Li', 'n_iters', 'flags', 'alpha', 'invL')}
        res['G'] = G.cpu().numpy()
        vb.close()
        return res

    ref, got = run(lens), run(with_empty)
    live = np.asarray(with_empty) > 0
    assert np.array_equal(got['gamma'], ref['gamma'])
    for k in ('pi', 'Li', 'n_iters', 'flags', 'G', 'alpha', 'invL'):
        assert np.array_equal(got[k][live], ref[k], equal_nan=True), k
    assert np.all(got['n_iters'][~live] == 0) and np.all(got['flags'][~live] == 0)
    assert np.all(np.isnan(got['Li'][~live]))
    assert np.all(got['G'][~live] == 0.0)
    assert np.all(got['pi'][~live] == np.float32(1.0 / S))
    assert np.all(got['alpha'][~live] == 0.0) and np.all(got['invL'][~live] == 0.0)    # as passed in (run() zeroes them)
    assert np.any(ref['flags'] & 4)               # the epsilon stop ended recordings: the float64 finishing phase ran
