"""NumPy restatement of the fused kernel's per-row link table (dks_fused.cuh, DESIGN.md 5.0.1): the build (domain, grid,
Chebyshev fit, float32 rounding of c2 .. c5, verification at the check points, one refinement) and the kernel's
evaluation, held to float64 L_s on a dense x grid.  CPU only."""
import numpy as np
import pytest

MARGIN, TOL, NODES = 33.0, 1e-9, 6
T = 0.5 - 0.5 * np.cos((2 * np.arange(NODES) + 1) * np.pi / (2 * NODES))
VINV = np.linalg.inv(np.vander(T, NODES, increasing=True))
CHECK = np.concatenate([[0.0], 0.5 * (T[:-1] + T[1:]), [1.0]])


def exact(x, ld, w, link):
    """float64 L_s(x) for the row's log2 Dm (ld) and weights w'_j = N w_j"""
    z = np.asarray(x, dtype=np.float64)[..., None] + ld
    e = np.exp2(-np.abs(z))
    r = w / (1.0 + e)
    s1 = np.where(z > 0, e * r, r).sum(-1)
    s0 = np.where(z > 0, r, e * r).sum(-1)
    return np.log(s1) - np.log(s0) if link == "logit" else s1 / ld.size


def poly(c, t):
    """interval coefficients c (float64 c0, c1; c2 .. c5 float32 values) at t in [0, 1]: float32 Horner tail, float64 head"""
    tf = t.astype(np.float32)
    c32 = c[..., 2:].astype(np.float32)
    q = c32[..., 0] + tf * (c32[..., 1] + tf * (c32[..., 2] + tf * c32[..., 3]))
    return c[..., 0] + t * (c[..., 1] + t * q.astype(np.float64))


def evaluate(tab, x_lo, h, x):
    """the kernel's evaluation: interval k and t from x, then the interval's polynomial"""
    v = (x - x_lo) / h
    k = np.floor(v).astype(np.int64)
    return poly(tab[k], v - k)


def build(ld, w, link):
    """(x_lo, h, table) as dks_set_shared_plan builds them, or None when the row fails verification at h = 1/8"""
    live = w > 0
    lmin, lmax = ld[live].min(), ld[live].max()
    for h in (0.25, 0.125):
        x_lo = np.floor((-MARGIN - lmax) / h) * h
        nint = int(np.ceil((MARGIN - lmin - x_lo) / h))
        x0 = x_lo + h * np.arange(nint)
        f = exact(x0[:, None] + h * T[None, :], ld, w, link)
        c = f @ VINV.T
        c[:, 2:] = c[:, 2:].astype(np.float32)
        xc = x0[:, None] + h * CHECK[None, :]
        err = np.abs(poly(c[:, None, :], np.broadcast_to(CHECK, xc.shape)) - exact(xc, ld, w, link))
        if err.max() <= TOL:
            return x_lo, h, c
    return None


def rows():
    rng = np.random.default_rng(7)
    out = {}
    d = rng.normal(0.0, 2.5, 100)
    out["bench_shaped"] = (d - np.rint(d.max()), np.ones(100))
    out["n1"] = (np.array([0.3]), np.ones(1))
    out["all_equal"] = (np.full(17, -0.4), np.ones(17))
    out["spread_100"] = (-100.0 * rng.random(64), np.ones(64))
    w = np.exp(rng.uniform(0, np.log(400.0), 50))
    w[[0, 7]] = [1.0, 400.0]
    w[3] = 0.0
    w = w / w.sum() * w.size
    d = rng.normal(0.0, 4.0, 50)
    out["skewed_weights"] = (d - np.rint(d.max()), w)
    return out


ROWS = rows()


@pytest.mark.parametrize("link", ["logit", "identity"])
@pytest.mark.parametrize("name", sorted(ROWS))
def test_table_holds_float64_link(name, link):
    ld, w = ROWS[name]
    built = build(ld, w, link)
    assert built is not None, "row fails verification at h = 1/8"
    x_lo, h, tab = built
    nint = tab.shape[0]
    rng = np.random.default_rng(1)
    x = np.concatenate([x_lo + h * (np.arange(nint)[:, None] + rng.random((nint, 16))).ravel(),
                        [x_lo, np.nextafter(x_lo + h * nint, -np.inf), x_lo + h * (nint - 1)]])
    x = x[(x - x_lo) / h < nint]                          # the kernel decides membership on v, as here
    err = np.abs(evaluate(tab, x_lo, h, x) - exact(x, ld, w, link))
    assert err.max() <= TOL, (name, link, h, err.max())


@pytest.mark.parametrize("link", ["logit", "identity"])
def test_beyond_the_domain_is_affine(link):
    """past either end of the domain L_s is affine to 1e-10, which is why the table stops there"""
    ld, w = ROWS["bench_shaped"]
    live = w > 0
    for x, dx in ((-MARGIN - ld[live].max(), -1.0), (MARGIN - ld[live].min(), 1.0)):
        xs = x + dx * np.array([0.0, 5.0, 10.0])
        y = exact(xs, ld, w, link)
        assert abs((y[2] - y[1]) - (y[1] - y[0])) < 2e-10


def test_n1_is_exactly_affine():
    """one background row: L_s(x) = -(x + log2 Dm) ln 2, the table reproduces it"""
    ld, w = ROWS["n1"]
    x_lo, h, tab = build(ld, w, "logit")
    x = np.linspace(x_lo, x_lo + h * tab.shape[0], 1001)[:-1]
    assert np.abs(evaluate(tab, x_lo, h, x) + (x + ld[0]) * np.log(2.0)).max() < 1e-11
