"""The wake layer's binary32 specification (oracle/wake.py and its companions) against the binary64 model written from
include/ocean.h (oracle/wake_model64.py), on the CPU.  The specification and the kernels were written together and are
bit-identical; this suite checks what they compute against the header's words: the ring index, the sponge ramp, the stencil
by orbit class, the edge zeros, the scroll, the sources at the exact cell centres, the foam update, blocked cells, the free
surface, the render map and the sample.

Every comparison is |spec - model| <= an a-priori per-cell bound, derived below (the bound functions), never a tolerance fitted
to the data.  Notation: u = 2^-24; hs(v) = half the binary32 spacing at |v|, the largest error of rounding a real v to
binary32 (round to nearest; hs(v) <= u |v| for normal v).  A binary32 operation on exact inputs a, b returns (a o b) + e with
|e| <= hs(a o b); with input errors da, db the result's error is the propagated one plus the rounding of the perturbed value.
Rounding is monotone, and max, min and the foam clamp are 1-Lipschitz, so they propagate an error without enlarging it."""
import numpy as np
import pytest
from scipy import ndimage

from oracle import wake as wk
from oracle import wake_coupling as wc
from oracle import wake_foam as wf
from oracle import wake_model64 as m64
from oracle import wake_obstacles as wo

U = 2.0 ** -24
TINY = 2.0 ** -149                      # the smallest binary32 spacing: one subnormal rounding
f32 = np.float32


def hs(v):
    """Half the binary32 spacing at |v| (binary64 array): bounds the rounding of v, or of anything within v's binade."""
    a = np.minimum(np.abs(np.asarray(v, np.float64)), 3.4e38).astype(np.float32)
    return 0.5 * np.spacing(a).astype(np.float64) * (1.0 + 2.0 ** -20)


def params(n, dx, damping, sponge_cells, sponge_damping):
    p = np.zeros((), wk.PARAMS)
    p["size"], p["cell_size"], p["damping"], p["sponge_cells"], p["sponge_damping"] = n, dx, damping, sponge_cells, sponge_damping
    return p


def largest_substep(dx) -> np.float32:
    """The largest binary32 sub-step the stability rule accepts at cell size dx."""
    h = np.float32(np.sqrt(float(np.float32(dx)) / wk.G))
    while not wk.stable(dx, h):
        h = np.nextafter(h, np.float32(0))
    while wk.stable(dx, np.nextafter(h, np.float32(np.inf))):
        h = np.nextafter(h, np.float32(np.inf))
    return h


# ---- the error bound of one sub-step ------------------------------------------------------------------------------------

def centre_error(src, states, tau):
    """Per source, a bound on |binary32 centre - binary64 centre| along x and z: cx = fl(x + fl(vx tau)), and for a body
    fl(cx + fl(pos + fl(lv tau))).  Adding an exact 0 is exact, so a source with vx tau = 0 carries no error there."""
    s = np.asarray(src).reshape(-1)
    out = []
    for ax, (p, v, q) in enumerate((("x", "vx", 0), ("z", "vz", 2))):
        t1 = s[v].astype(np.float64) * tau
        a = s[p].astype(np.float64) + t1
        e = hs(t1) + np.where(t1 != 0, hs(np.abs(a) + hs(t1)), 0.0)
        att = (s["body"] >= 0) & (s["body"] < (0 if states is None else len(states)))
        for k in np.flatnonzero(att):
            b = states[s["body"][k]]
            t2 = float(b["linear_velocity"][q]) * tau
            bb = float(b["position"][q]) + t2
            e2 = hs(t2) + (hs(abs(bb)) if t2 != 0 else 0.0)
            e[k] = e[k] + e2 + hs(abs(a[k] + bb) + e[k] + e2)
        out.append(e)
    return out


def speed2_error(src, states):
    """Per source, (|v|^2 exact, a bound on the binary32 |v|^2's error): v = fl(vx + lv) for a body, fl(fl(vx vx) + fl(vz vz))."""
    s = np.asarray(src).reshape(-1)
    vx, vz = s["vx"].astype(np.float64), s["vz"].astype(np.float64)
    dvx, dvz = np.zeros(len(s)), np.zeros(len(s))
    att = (s["body"] >= 0) & (s["body"] < (0 if states is None else len(states)))
    for k in np.flatnonzero(att):
        b = states[s["body"][k]]
        vx[k] += float(b["linear_velocity"][0])
        vz[k] += float(b["linear_velocity"][2])
        dvx[k], dvz[k] = hs(vx[k]), hs(vz[k])
    ex = 2 * np.abs(vx) * dvx + dvx ** 2
    ex = ex + hs(vx * vx + ex)
    ez = 2 * np.abs(vz) * dvz + dvz ** 2
    ez = ez + hs(vz * vz + ez)
    v2 = vx * vx + vz * vz
    return v2, ex + ez + hs(v2 + ex + ez)


def footprint_bound(M, src, states, tau):
    """(phi, sigma, ephi, esigma) [N][N]: the model's binary64 phi and sigma at the exact cell centres and bounds on the
    binary32 specification's error, which comes from
      * the centres: the corner x0 = (float)((double)ox dx) is |x0 - ox dx| off, then fl(x0 + fl((i + 1/2) dx));
      * the source centres (centre_error);
      * ex = fl(px - cx), d2 = fl(fl(ex ex) + fl(ez ez)), r2 = fl(r r), q = fl(d2 / r2), w = fl(1 - q), fl(w w),
        fl(head ww) (fl(ww |v|^2)), each propagated to first order with the squares' second-order terms kept;
      * the test d2 < r2: a cell the two classify differently has |w| within the bound of w, so head w^2 <= head 4 Dw^2,
        which the term 4 Dw^2 covers;
      * the sum over the m sources at a cell, in index order: at most m roundings of partial sums <= sum |phi_k|."""
    n, dx = M.n, float(f32(M.cell_size))
    px, pz = m64.cell_centres(n, dx, M.origin)
    x0, z0 = m64.corner(M.origin, dx)
    y = (np.arange(n) + 0.5) * dx
    dpx = abs(x0 - float(M.origin[0]) * dx) + hs(y) + hs(np.abs(x0 + y) + hs(y)) + 2.0 ** -52 * np.abs(px)
    dpz = abs(z0 - float(M.origin[1]) * dx) + hs(y) + hs(np.abs(z0 + y) + hs(y)) + 2.0 ** -52 * np.abs(pz)
    cx, cz, r, head, v2, valid = m64.source_terms(src, states, tau)
    dcx, dcz = centre_error(src, states, tau)
    v2x, dv2 = speed2_error(src, states)
    phi, sig = np.zeros((n, n)), np.zeros((n, n))
    ephi, esig = np.zeros((n, n)), np.zeros((n, n))
    aphi, asig, cnt = np.zeros((n, n)), np.zeros((n, n)), np.zeros((n, n))
    for k in np.flatnonzero(valid):
        ex = px - cx[k]
        ez = pz - cz[k]
        Ex = dpx + dcx[k] + hs(np.abs(ex) + dpx + dcx[k])
        Ez = dpz + dcz[k] + hs(np.abs(ez) + dpz + dcz[k])
        r2, Dr2 = r[k] * r[k], hs(r[k] * r[k])
        # only cells that may be inside for either form: d2 - Dd < r2 + Dr2
        xs = np.flatnonzero(np.abs(ex) - Ex < r[k] * 1.001 + Ex)
        zs = np.flatnonzero(np.abs(ez) - Ez < r[k] * 1.001 + Ez)
        if not len(xs) or not len(zs):
            continue
        X, EX = ex[xs][None, :], Ex[xs][None, :]
        Z, EZ = ez[zs][:, None], Ez[zs][:, None]
        Exx = 2 * np.abs(X) * EX + EX ** 2
        Exx = Exx + hs(X * X + Exx)
        Ezz = 2 * np.abs(Z) * EZ + EZ ** 2
        Ezz = Ezz + hs(Z * Z + Ezz)
        d2 = X * X + Z * Z
        Dd = Exx + Ezz + hs(d2 + Exx + Ezz)
        q = d2 / r2
        q_hi = (d2 + Dd) / (r2 - Dr2)
        q_lo = np.maximum(d2 - Dd, 0) / (r2 + Dr2)
        Dq = np.maximum(q_hi - q, q - q_lo) + hs(q_hi)
        near = q - Dq < 1.0
        w = np.where(q < 1.0, 1.0 - q, 0.0)
        Dw = Dq + hs(np.abs(1.0 - q) + Dq)
        ww = w * w
        Dww = 2 * w * Dw + 4 * Dw * Dw
        Dww = Dww + hs(ww + Dww)
        Dp = abs(head[k]) * Dww + hs(abs(head[k]) * (ww + Dww))
        Ds = v2x[k] * Dww + (ww + Dww) * dv2[k] + hs((ww + Dww) * (v2x[k] + dv2[k]))
        sl = np.ix_(zs, xs)
        phi[sl] += head[k] * ww
        sig[sl] += v2x[k] * ww
        ephi[sl] += np.where(near, Dp, 0.0)
        esig[sl] += np.where(near, Ds, 0.0)
        aphi[sl] += np.where(near, abs(head[k]) * ww + Dp, 0.0)
        asig[sl] += np.where(near, v2x[k] * ww + Ds, 0.0)
        cnt[sl] += near
    ephi = (ephi + cnt * (U * aphi + TINY)) * (1 + 1e-6)
    esig = (esig + cnt * (U * asig + TINY)) * (1 + 1e-6)
    return phi, sig, ephi, esig


def substep_bound(tr, M, dx, eh_in, ehp_in, ephi, esig, ef_in=None):
    """Bounds on |h_new| and |F'| of the binary32 specification against the model, from the input errors eh_in, ehp_in,
    ef_in of its h, h_prev and F and the footprint's ephi, esig:
      s = fl(h + phi)                           es = eh + ephi + hs(|h + phi| + eh + ephi)            (0 on blocked cells)
      c = the 28-class sum                      ec = |G| * es + 169 u |G| * (|s| + es)
          (169 terms: every term passes through at most 36 roundings -- one tap product, seven orbit additions and 28
          accumulations -- so (number of additions + 1) u = 169 u times sum |G| |s| bounds the summation, with margin)
      a1, a2, a3 rounded once                   da = hs(a)
      h_new = fl(fl(fl(a1 h) - fl(a2 h_prev)) - fl(a3 c)): three products, two differences, each with its rounding
      beta = fl(c / dx), b = max(fl(beta - whitecap), 0), x = fl(fl(F d) + fl(fl(gh b) + fl(sh sigma))), F' = clamp(x, 0, 1)."""
    a1, a2, a3 = tr["a"]
    h, hp, c, s, B = tr["h"], tr["h_prev"], tr["c"], tr["s"], tr["B"]
    absk = np.abs(M.k)
    es = eh_in + ephi + hs(np.abs(s) + eh_in + ephi)
    es = np.where(B, 0.0, es)
    corr = lambda f: ndimage.correlate(f, absk, mode="constant", cval=0.0)
    ec = corr(es) + 169 * U * corr(np.abs(s) + es) + 169 * TINY
    e1 = hs(a1) * (np.abs(h) + eh_in) + np.abs(a1) * eh_in
    e1 = e1 + hs(np.abs(a1 * h) + e1)
    e2 = hs(a2) * (np.abs(hp) + ehp_in) + np.abs(a2) * ehp_in
    e2 = e2 + hs(np.abs(a2 * hp) + e2)
    e3 = np.abs(a3) * ec + hs(a3) * (np.abs(c) + ec)
    e3 = e3 + hs(np.abs(a3 * c) + e3)
    d1 = a1 * h - a2 * hp
    e4 = e1 + e2 + hs(np.abs(d1) + e1 + e2)
    hn = d1 - a3 * c
    eh = (e4 + e3 + hs(np.abs(hn) + e4 + e3)) * (1 + 1e-6)
    eh = np.where(B, 0.0, eh)
    if "x" not in tr:
        return eh, None, ec
    F, d, gh, sh, b, x = tr["F"], tr["d"], tr["gh"], tr["sh"], tr["b"], tr["x"]
    ef_in = np.zeros_like(F) if ef_in is None else ef_in
    beta = c / dx
    eb = ec / dx + hs(np.abs(beta) + ec / dx)
    eb = eb + hs(np.abs(b) + eb)                       # max(., 0) is 1-Lipschitz: no threshold to exclude
    bp = np.maximum(b, 0.0)
    t1 = d * ef_in + hs(np.abs(F * d) + d * ef_in)
    t2 = gh * eb + hs(gh * (bp + eb))
    t3 = sh * esig + hs(sh * (tr["sigma"] + esig))
    t4 = t2 + t3 + hs(gh * bp + sh * tr["sigma"] + t2 + t3)
    ex = (t1 + t4 + hs(np.abs(x) + t1 + t4)) * (1 + 1e-6)
    return eh, np.where(B, 0.0, ex), ec           # the clamp to [0, 1] is 1-Lipschitz: F' is within ex as x is


# ---- one scene: the specification and the model from the same binary32 state ----------------------------------------------

def edge_sources(rng, n, dx, k, origin, states=None):
    """Sources spread over the window and straddling all four edges, some moving, some on bodies."""
    s = np.zeros(k, wk.SOURCE)
    ext = n * dx
    x0, z0 = origin[0] * dx, origin[1] * dx
    s["x"] = x0 + rng.uniform(-0.05, 1.05, k) * ext
    s["z"] = z0 + rng.uniform(-0.05, 1.05, k) * ext
    s["x"][:4] = x0 + np.array([0.0, ext, 0.3 * ext, 0.7 * ext])        # centres on the edges
    s["z"][:4] = z0 + np.array([0.4 * ext, 0.6 * ext, 0.0, ext])
    s["vx"], s["vz"] = rng.uniform(-3, 3, k), rng.uniform(-3, 3, k)
    s["radius"] = rng.uniform(2, 12, k) * dx
    s["head"] = rng.uniform(-0.4, 0.4, k)
    s["body"] = -1
    if states is not None:
        att = rng.random(k) < 0.3
        s["body"][att] = rng.integers(0, len(states), att.sum())
        s["x"][att], s["z"][att] = rng.uniform(-2, 2, att.sum()), rng.uniform(-2, 2, att.sum())
    s["head"][5], s["radius"][6] = np.nan, 0.0                            # contribute nothing
    return s


def run_scene(n, dx, damping, sponge_cells, sponge_damping, *, substeps=1, scroll=(0, 0), origin=(0, 0), foam=None, mask=None,
              mask_origin=(0, 0), sources=8, seed=0, h_scale=0.05, big_origin_sources=False):
    """Random h, h_prev (and F) at `origin`; one call of `substeps` sub-steps at the largest accepted sub-step, scrolled by
    `scroll`, on the specification and on the model; the propagated bound.  Returns (spec layer, model, bound on h, on F,
    trace, dt, sources, states)."""
    rng = np.random.default_rng(seed)
    p = params(n, dx, damping, sponge_cells, sponge_damping)
    L = wo.Layer(p, wf.foam_params(**foam) if foam else None)
    L.foam_on = foam is not None
    M = m64.Model(p, None if foam is None else (foam["whitecap"], foam["grow_rate"], foam["stir_rate"], foam["decay_rate"]),
                  mask, mask_origin)
    if mask is not None:
        L.set_obstacles(mask, mask_origin)
    h0 = (rng.standard_normal((n, n)) * h_scale).astype(np.float32)
    hp0 = (h0 + rng.standard_normal((n, n)).astype(np.float32) * f32(h_scale / 10)).astype(np.float32)
    L.h, L.h_prev, L.origin = h0.copy(), hp0.copy(), tuple(origin)
    M.h, M.h_prev, M.origin = h0.astype(np.float64), hp0.astype(np.float64), tuple(origin)
    if foam is not None:
        F0 = rng.uniform(0, 1, (n, n)).astype(np.float32)
        F0[rng.random((n, n)) < 0.2] = 0.0
        L.foam, M.F = F0.copy(), F0.astype(np.float64)
    states = np.zeros(3, wk.STATE)
    new_origin = (origin[0] + scroll[0], origin[1] + scroll[1])
    states["position"] = rng.uniform(0, n * dx, (3, 3)) + np.array([new_origin[0] * dx, 0, new_origin[1] * dx])
    states["linear_velocity"] = rng.uniform(-2, 2, (3, 3))
    src = edge_sources(rng, n, dx, sources, new_origin, states)
    hmax = largest_substep(dx)
    dt = float(hmax) * substeps
    wo.step(L, None, dt, substeps, new_origin, src, states)
    eh, ef, trace = model_call(M, dt, substeps, new_origin, src, states)
    return L, M, eh, ef, trace, dt, src, states


def model_call(M, dt, substeps, origin, src, states):
    """One step call of the model from its binary32 start state, with the bound on the binary32 result propagated over the
    sub-steps: (bound on h, bound on F, trace).  The start state is exact in both, so the first sub-step's input errors are 0
    (on a scrolled first sub-step too: the scroll moves values without rounding them)."""
    trace = []
    M.step(dt, substeps, origin, src, states, trace)
    n = M.n
    eh, ehp, ef = np.zeros((n, n)), np.zeros((n, n)), np.zeros((n, n))
    for tr in trace:
        ephi, esig = footprint_bound(M, src, states, tr["tau"])[2:] if src is not None and len(src) else (0.0, 0.0)
        new_eh, new_ef, _ = substep_bound(tr, M, float(f32(M.cell_size)), eh, ehp, ephi, esig, ef)
        eh, ehp = new_eh, eh
        if new_ef is not None:
            ef = new_ef
    return eh, ef, trace


def check(L, M, eh, ef, what, max_ratio_to_h=1e-3):
    err = np.abs(L.h.astype(np.float64) - M.h)
    assert np.all(np.isfinite(M.h)) and np.all(np.isfinite(eh))
    ratio = float(np.max(np.where(eh > 0, err / np.maximum(eh, 1e-300), np.where(err > 0, np.inf, 0.0))))
    scale = float(np.abs(M.h).max())
    print(f"{what}: h max |spec - model| / bound = {ratio:.3f}, bound max {eh.max():.3g} = {eh.max() / scale:.2e} of max|h| {scale:.3g}")
    assert np.all(err <= eh), (what, np.argwhere(err > eh)[:5], ratio)
    assert eh.max() <= max_ratio_to_h * scale, (what, eh.max(), scale)       # the bound is not vacuous
    if L.foam_on:
        errf = np.abs(L.foam.astype(np.float64) - M.F)
        excluded = 0                                    # max(., 0) and the clamp are 1-Lipschitz: nothing to exclude
        rf = float(np.max(np.where(ef > 0, errf / np.maximum(ef, 1e-300), np.where(errf > 0, np.inf, 0.0))))
        print(f"{what}: F max |spec - model| / bound = {rf:.3f}, bound max {ef.max():.3g}, {excluded} cells excluded")
        assert np.all(errf <= ef), (what, np.argwhere(errf > ef)[:5], rf)
        assert ef.max() <= max_ratio_to_h and 0.01 < M.F.mean() < 0.99       # F lies in [0, 1]
    return ratio


FOAM = dict(whitecap=0.02, grow_rate=3.0, stir_rate=0.5, decay_rate=0.7)


@pytest.mark.parametrize("sponge_cells", [0, 1, 63, 64])
@pytest.mark.parametrize("dx", [0.25, 1.0])
@pytest.mark.parametrize("damping,sponge_damping", [(0.05, 2.0), (3.0, 0.5)])
def test_one_call_at_128_every_sponge_width(sponge_cells, dx, damping, sponge_damping):
    """N = 128 (64 = N/2: the window is all sponge), S = 1 at the largest sub-step, damping above and below sponge_damping,
    foam on, sources straddling the window's edges; every ring of the coefficient table is used."""
    L, M, eh, ef, tr, *_ = run_scene(128, dx, damping, sponge_cells, sponge_damping, foam=FOAM, seed=sponge_cells + int(4 * dx))
    check(L, M, eh, ef, f"N=128 sponge={sponge_cells} dx={dx} damping={damping}/{sponge_damping}")


def test_rings_are_distinguished():
    """The bound resolves a one-ring shift of the coefficient table: the model with the ring index min(edge + 1, sponge_cells)
    is outside the bound near the edge."""
    L, M, eh, ef, tr, dt, src, st = run_scene(128, 1.0, 0.05, 63, 2.0, seed=5)
    a1, a2, a3 = tr[0]["a"]
    h = m64.substep(dt, 1)
    n = 128
    i = np.arange(n)
    e = np.minimum(i, n - 1 - i)
    ring = np.minimum(np.minimum(e[None, :], e[:, None]) + 1, 63)
    t = (63 - ring) / 63
    alpha = np.where(ring < 63, 0.05 + (2.0 - 0.05) * t * t, 0.05)
    ah = alpha * h
    b1, b2, b3 = (2 - ah) / (1 + ah), 1 / (1 + ah), wk.G * h * h / (1.0 * (1 + ah))
    wrong = (b1 * tr[0]["h"] - b2 * tr[0]["h_prev"]) - b3 * tr[0]["c"]
    assert np.mean(np.abs(L.h - wrong) > eh) > 0.5


@pytest.mark.parametrize("sponge_cells", [1, 64])
def test_one_call_at_2048(sponge_cells):
    """N = 2048, foam on, a scrolled first sub-step (3, -2), at the largest sub-step."""
    L, M, eh, ef, *_ = run_scene(2048, 0.25, 0.1, sponge_cells, 1.0, foam=FOAM, scroll=(3, -2), sources=8, seed=2048 + sponge_cells)
    check(L, M, eh, ef, f"N=2048 sponge={sponge_cells}")


def test_blocked_cells_and_a_scroll_across_the_mask():
    """An obstacle mask with single blocked cells next to open ones and a wall, the window scrolled by (5, -7) over it."""
    n = 128
    rng = np.random.default_rng(3)
    mask = (rng.random((n + 40, n + 40)) < 0.05).astype(np.uint8)
    mask[60:64, :] = 1
    L, M, eh, ef, *_ = run_scene(n, 0.25, 0.05, 24, 3.0, foam=FOAM, scroll=(5, -7), mask=mask, mask_origin=(-20, -15), seed=9)
    B = m64.blocked(mask, (-20, -15), M.origin, n)
    assert B.any() and not B.all()
    assert not L.h[B].any() and not M.h[B].any()
    check(L, M, eh, ef, "blocked cells, scrolled (5, -7)")


def test_three_sub_steps_with_the_propagated_bound():
    """S = 3: the bound of each sub-step takes the previous sub-step's bound as its input error on h (and h_prev), so it
    holds for the whole call; it grows by about |a1| + |a2| + |a3| sum|G| per sub-step, still small after three."""
    L, M, eh, ef, *_ = run_scene(128, 1.0, 0.2, 16, 1.5, foam=FOAM, substeps=3, scroll=(-4, 9), seed=33)
    check(L, M, eh, ef, "S=3 propagated", max_ratio_to_h=1e-2)


def test_free_surface_render_map_and_sample():
    """e = h + phi_end at tau_end = (float)S h; the render map's binary32 central differences and halves; the bilinear
    sample, on and just beyond the four edges (points within the sample's position bound of an edge are counted and
    excluded: the sample is discontinuous there)."""
    n, dx = 128, 0.25
    mask = np.zeros((n, n), np.uint8)
    mask[30:40, 50:90] = 1
    L, M, eh, ef, tr, dt, src, st = run_scene(n, dx, 0.05, 8, 1.0, mask=mask, mask_origin=(0, 0), origin=(-11, 6), seed=12)
    # the free surface of the spec's h (so the comparison isolates phi_end and the addition)
    e32 = wo.free_surface(L, src, st, dt, 1)
    M.h = L.h.astype(np.float64)
    e64 = M.free_surface(dt, 1, src, st)
    tau = float(f32(1) * m64.substep(dt, 1))
    _, _, ephi, _ = footprint_bound(M, src, st, tau)
    B = m64.blocked(mask, (0, 0), M.origin, n)
    be = np.where(B, 0.0, ephi + hs(np.abs(e64) + ephi))
    assert np.all(np.abs(e32 - e64) <= be) and np.abs(e64).max() > 0.01
    # render map: gx = fl(fl(h[i+1] - h[i-1]) / fl(2 dx)) (2 dx exact), then rounded to half
    m = L.render_map().astype(np.float64)
    ref = m64.render_map(L.h, dx)
    g = np.abs(ref[..., 1:3])
    eg = hs(g * 2 * dx) / (2 * dx)
    eg = eg + hs(g + eg)
    hs16 = lambda v: np.maximum(2.0 ** -11 * np.abs(v), 2.0 ** -25)
    assert np.all(np.abs(m[..., 0] - ref[..., 0]) <= hs16(ref[..., 0]))
    assert np.all(np.abs(m[..., 1:3] - ref[..., 1:3]) <= eg + hs16(g + eg))
    # the sample: u = fl(fl(fl(x - x0) / dx) - 0.5) against x / dx - ox - 0.5
    rng = np.random.default_rng(4)
    x0, z0 = m64.corner(M.origin, dx)
    ext = n * dx
    pts = np.concatenate([rng.uniform([x0 - 1, z0 - 1], [x0 + ext + 1, z0 + ext + 1], (400, 2)),
                          [[x0, z0 + 3], [x0 + ext, z0 + 3], [x0 + 3, z0], [x0 + 3, z0 + ext],
                           [np.nextafter(f32(x0), f32(-1e9)), z0 + 3], [x0 + 5, np.nextafter(f32(z0 + ext), f32(-1e9))]]])
    pts = pts.astype(np.float32)
    s32, s64 = L.sample(pts), m64.sample(L.h, dx, M.origin, pts.astype(np.float64))
    gx, gz = m64.gradients(L.h, dx)
    fm = [np.abs(L.h).max(), np.abs(gx).max(), np.abs(gz).max()]
    xs = pts.astype(np.float64)
    du = (hs(xs - np.array([x0, z0])) + np.abs(np.array([x0, z0]) - np.array(M.origin) * dx)) / dx
    du = du + hs(np.abs(xs - np.array([x0, z0])) / dx + du) + hs(np.abs(xs - np.array([x0, z0])) / dx + 0.5 + du)
    du = du + hs(1.0)                                   # fu = fl(u - floor(u))
    uu = xs / dx - np.array(M.origin) - 0.5
    edge = np.any((np.abs(uu + 0.5) <= du) | (np.abs(uu - (n - 0.5)) <= du), axis=1)
    excluded = int(edge.sum())
    print(f"sample: {excluded} of {len(pts)} points within the position bound of an edge")
    assert excluded <= 8
    for k in np.flatnonzero(~edge):
        for f in range(3):
            bound = 2 * fm[f] * (du[k, 0] + du[k, 1]) * (1 + 1e-3) + 12 * U * fm[f] + TINY
            assert abs(s32[k, f] - s64[k, f]) <= bound, (k, f, s32[k, f], s64[k, f], bound)


def test_far_origin_position_error_is_bounded():
    """At a window ~2^24 cells from the world origin, with a cell size that makes the corner inexact, the binary32 centres
    are within the position bound -- and the bound resolves the corner of (float)ox * dx, 1 ulp of x0 off, at most cells."""
    dx = 1.9921875                                     # 255 / 128: (i + 1/2) dx exact, ox dx within 0.008 of a binary32
    origin = (2 ** 24 + 1, -(2 ** 24 + 1))
    L, M, eh, ef, tr, dt, src, st = run_scene(128, dx, 0.05, 8, 1.0, origin=origin, sources=8, seed=21, h_scale=0.0)
    # zero start state: h is driven by phi alone, so the whole bound is the footprint's
    err = np.abs(L.h.astype(np.float64) - M.h)
    assert np.all(err <= eh) and np.abs(M.h).max() > 1e-3
    px, _ = m64.cell_centres(128, dx, origin)
    x0h = m64.corner(origin, dx)[0]
    p32 = (f32(x0h) + (np.arange(128, dtype=np.float32) + f32(0.5)) * f32(dx)).astype(np.float64)
    x0m = float(f32(float(f32(origin[0])) * dx))       # (float)ox * dx
    pm = (f32(x0m) + (np.arange(128, dtype=np.float32) + f32(0.5)) * f32(dx)).astype(np.float64)
    y = (np.arange(128) + 0.5) * dx
    dpx = abs(x0h - origin[0] * dx) + hs(y) + hs(np.abs(x0h + y) + hs(y))
    print(f"far origin: centre error max {np.abs(p32 - px).max():.3f} m = {np.abs(p32 - px).max() / dx:.3f} cells, "
          f"bound {dpx.max():.3f} m; with (float)ox * dx {np.abs(pm - px).max():.3f} m")
    assert np.all(np.abs(p32 - px) <= dpx)
    assert x0m != x0h and np.mean(np.abs(pm - px) > dpx) > 0.5


def test_bounding_box_rasterisation_is_byte_identical():
    """wake.rasterise with its footprint box and without, on random scenes: sources straddling the box and the window's
    edges, tiny and huge radii, far and inexact corners, an infinite corner, centres at +-FLT_MAX."""
    rng = np.random.default_rng(17)
    for trial in range(12):
        n = 128
        dx = f32([0.25, 1.0, 0.1, 1e-3, 1e20, 1.9921875][trial % 6])
        origin = [(0, 0), (-7, 13), (2 ** 31 + 3, -(2 ** 31) - 2), (2 ** 40, -(2 ** 40)), (2 ** 63 - 100, -(2 ** 63)),
                  (12345, 54321)][trial // 2]
        x0, z0 = wk.world_origin(origin, dx)
        ext = float(n * dx)
        k = 60
        s = np.zeros(k, wk.SOURCE)
        with np.errstate(all="ignore"):
            s["x"] = (float(x0) + rng.uniform(-0.2, 1.2, k) * ext) if np.isfinite(x0) else rng.uniform(-1e3, 1e3, k)
            s["z"] = (float(z0) + rng.uniform(-0.2, 1.2, k) * ext) if np.isfinite(z0) else rng.uniform(-1e3, 1e3, k)
        s["vx"], s["vz"] = rng.uniform(-3, 3, k), rng.uniform(-3, 3, k)
        s["radius"] = rng.choice([0.3, 1.0, 5.0, 40.0], k) * dx
        s["head"] = rng.uniform(-1, 1, k)
        s["body"] = -1
        s["x"][0], s["radius"][1], s["x"][2] = 3.0e38, 1e19, -3.4e38
        st = np.zeros(0, wk.STATE)
        tau = f32(rng.uniform(0, 1)) * f32(dx)
        full = wk.rasterise(n, dx, origin, s, st, tau, box=False)
        boxed = wk.rasterise(n, dx, origin, s, st, tau, box=True)
        assert full.tobytes() == boxed.tobytes(), trial
