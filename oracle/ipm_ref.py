"""ORACLE (test infrastructure only -- never imported by the product path).

Generic primal-dual interior-point NLP solver: a restatement of the published
Ipopt algorithm (Waechter & Biegler, Math. Prog. 106(1), 2006 -- the solver the
reference calls at ParkingSignedDist.jl:41-43,240; Ipopt itself is an
un-vendored dependency and is not installed here, so this is the "IPOPT
stand-in", not IPOPT).  Linear algebra is deliberately generic and dense
(LAPACK dsytrf Bunch-Kaufman LDL' of the full augmented KKT matrix, inertia read
from the factor) so that it is independent of the stage-structured
Riccati/Schur elimination used by the CUDA solver.

Formulation:  min f(z) s.t. cE(z)=0, g(z)-s=0, gL<=s<=gU, zL<=z<=zU.
One multiplier pair (vL,vU) per slack; the row multiplier is yI = vU - vL.

Options mirrored from the reference call site: tol=1e-5, max_iter=200,
min_hessian_perturbation=1e-12, jacobian_regularization_value=1e-7,
alpha_for_y=min (ParkingSignedDist.jl:41-43).  Everything else = Ipopt default.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np
import scipy.sparse as sps
from scipy.linalg import lapack


@dataclass
class IpmOptions:
    tol: float = 1e-5
    max_iter: int = 200
    mu_init: float = 0.1
    mu_min_factor: float = 0.1          # mu_min = tol * factor  (Ipopt: tol/10)
    kappa_eps: float = 10.0
    kappa_mu: float = 0.2
    theta_mu: float = 1.5
    tau_min: float = 0.99
    kappa1: float = 1e-2                # bound_push
    kappa2: float = 1e-2                # bound_frac
    kappa_sigma: float = 1e10
    s_max: float = 100.0
    dual_inf_tol: float = 1.0
    constr_viol_tol: float = 1e-4
    compl_inf_tol: float = 1e-4
    # inertia correction
    dw_min: float = 1e-12               # min_hessian_perturbation (reference option)
    dw_first: float = 1e-4
    dw_max: float = 1e20
    kw_minus: float = 1.0 / 3.0
    kw_plus: float = 8.0
    kw_plus_first: float = 100.0
    # filter line search
    gamma_theta: float = 1e-5
    gamma_phi: float = 1e-8
    delta: float = 1.0
    s_theta: float = 1.1
    s_phi: float = 2.3
    eta_phi: float = 1e-8
    gamma_alpha: float = 0.05
    max_backtrack: int = 40
    # always-on dual regularisation for selected equality rows (see DESIGN.md "KKT solve")
    dc_rows: np.ndarray | None = None   # boolean mask over equality rows
    dc_value: float = 1e-9
    verbose: bool = False
    # "dense": LAPACK dsytrf (Bunch-Kaufman) on the dense KKT matrix -- the validation path.
    # "sparse": SuperLU in symmetric mode with diagonal pivoting (K = L D L', inertia = signs of D by Sylvester's
    #           law); falls back to "dense" whenever SuperLU had to pivot off the diagonal or the solve residual is
    #           poor.  This is the generic sparse-direct path (what Ipopt does with MUMPS) used for CPU timing.
    linsolve: str = "dense"
    order: np.ndarray | None = None     # symmetric ordering of the (n + mE) KKT unknowns for the sparse path
    max_kick: int = 3                   # restoration substitute: barrier kicks after a failed line search
    freeze_degenerate: float = 0.0      # > 0: an always-regularised row whose Jacobian row is below this threshold
                                        # keeps its multiplier this iteration (its linearisation carries no information;
                                        # Newton on |p|^2 = 1 from p = 0, QuadcopterSignedDist.jl:169 with l = 0.05)
    # index arrays of variables that a solver may carry as ONE variable (the time scale tied by the chain rows
    # timeScale[k] == timeScale[k+1], which the CUDA solver eliminates, DESIGN.md section 3): their dual residuals count as one
    # entry, their sum -- the dual infeasibility of the eliminated formulation.  The Newton steps of the two formulations are
    # the same; only the optimality error, and so the barrier updates and the stopping test, differ.
    dual_sum_groups: list | None = None
    snapshots: tuple = ()               # iteration counts K at which IpmResult.snaps[K] keeps the primal z: the z that a run
                                        # with max_iter = K returns, so one run pins several K


@dataclass
class IpmResult:
    z: np.ndarray
    s: np.ndarray
    yE: np.ndarray
    vL: np.ndarray
    vU: np.ndarray
    zLm: np.ndarray
    zUm: np.ndarray
    status: int                 # 1 converged, 0 max_iter, -1 line-search failure, -2 inertia failure
    iters: int
    err: float
    mu: float
    log: list = field(default_factory=list)
    snaps: dict = field(default_factory=dict)


class _SparseLDL:
    """SuperLU, symmetric mode, diagonal pivots only -> K = P'(L D L')P ; inertia from sign(diag(U))."""

    def __init__(self, K, order=None):
        from scipy.sparse.linalg import splu
        self.order = order
        self.K = K.tocsc() if order is None else K.tocsr()[order][:, order].tocsc()
        self.ok = False
        try:
            self.lu = splu(self.K, permc_spec="NATURAL" if order is not None else "MMD_AT_PLUS_A",
                           diag_pivot_thresh=0.0, options=dict(SymmetricMode=True))
        except RuntimeError:
            return
        if not np.array_equal(self.lu.perm_r, self.lu.perm_c):
            return
        d = self.lu.U.diagonal()
        self.npos = int((d > 0).sum()); self.nneg = int((d < 0).sum()); self.nzero = int((d == 0).sum())
        self.ok = True

    def solve(self, rhs):
        if self.order is not None:
            rhs = rhs[self.order]
        x = self._solve(rhs)
        if self.order is not None:
            y = np.empty_like(x); y[self.order] = x
            return y
        return x

    def _solve(self, rhs):
        x = self.lu.solve(rhs)
        for _ in range(2):
            x = x + self.lu.solve(rhs - self.K @ x)
        self.resid = np.abs(rhs - self.K @ x).max() / max(1.0, np.abs(rhs).max())
        return x


def _push(x, lo, hi, k1, k2):
    """Ipopt initial-point projection (section 3.6 of the paper)."""
    x = x.copy()
    lo = np.where(np.isfinite(lo), lo, -1e300); hi = np.where(np.isfinite(hi), hi, 1e300)
    both = (lo > -1e299) & (hi < 1e299)
    pl = np.where(both, np.minimum(k1 * np.maximum(1, np.abs(lo)), k2 * (hi - lo)), k1 * np.maximum(1, np.abs(lo)))
    pu = np.where(both, np.minimum(k1 * np.maximum(1, np.abs(hi)), k2 * (hi - lo)), k1 * np.maximum(1, np.abs(hi)))
    fl = lo > -1e299; fu = hi < 1e299
    x[fl] = np.maximum(x[fl], (lo + pl)[fl])
    x[fu] = np.minimum(x[fu], (hi - pu)[fu])
    return x


def _ldl_inertia(K):
    """Bunch-Kaufman factorisation; returns (factor, ipiv, n_pos, n_neg, n_zero)."""
    ldu, ipiv, info = lapack.dsytrf(K, lower=1)
    if info < 0:
        raise RuntimeError("dsytrf argument error")
    n = K.shape[0]
    npos = nneg = nzero = 0
    i = 0
    d = np.diag(ldu)
    while i < n:
        if ipiv[i] > 0:
            if d[i] > 0: npos += 1
            elif d[i] < 0: nneg += 1
            else: nzero += 1
            i += 1
        else:
            a, b_, c = ldu[i, i], ldu[i + 1, i], ldu[i + 1, i + 1]
            det = a * c - b_ * b_
            tr = a + c
            if det < 0: npos += 1; nneg += 1
            elif det > 0:
                if tr > 0: npos += 2
                else: nneg += 2
            else: nzero += 1; npos += (tr > 0); nneg += (tr < 0)
            i += 2
    if info > 0:
        nzero = max(nzero, 1)
    return ldu, ipiv, npos, nneg, nzero


def solve(nlp, z0, opt: IpmOptions | None = None, yE0=None) -> IpmResult:
    o = opt or IpmOptions()
    n, mE, mI = nlp.n, nlp.mE, nlp.mI
    zL, zU, gL, gU = nlp.zL, nlp.zU, nlp.gL, nlp.gU
    hasL, hasU = np.isfinite(zL), np.isfinite(zU)
    sHasL, sHasU = np.isfinite(gL), np.isfinite(gU)
    dc = np.zeros(mE)
    if o.dc_rows is not None:
        dc[o.dc_rows] = o.dc_value

    z = _push(np.asarray(z0, float), zL, zU, o.kappa1, o.kappa2)
    s = _push(nlp.g(z), gL, gU, o.kappa1, o.kappa2)
    yE = np.zeros(mE) if yE0 is None else yE0.copy()
    zLm = np.where(hasL, 1.0, 0.0); zUm = np.where(hasU, 1.0, 0.0)
    vL = np.where(sHasL, 1.0, 0.0); vU = np.where(sHasU, 1.0, 0.0)
    mu = o.mu_init
    tau = max(o.tau_min, 1 - mu)
    mu_min = o.tol * o.mu_min_factor
    n_mult = mE + mI + hasL.sum() + hasU.sum() + sHasL.sum() + sHasU.sum()
    n_bmult = hasL.sum() + hasU.sum() + sHasL.sum() + sHasU.sum()

    def gaps(z, s):
        return (np.where(hasL, z - zL, 1.0), np.where(hasU, zU - z, 1.0),
                np.where(sHasL, s - gL, 1.0), np.where(sHasU, gU - s, 1.0))

    def theta(z, s):
        return np.abs(nlp.cE(z)).sum() + np.abs(nlp.g(z) - s).sum()

    def phi(z, s, mu):
        a, b_, c, d = gaps(z, s)
        if (a <= 0).any() or (b_ <= 0).any() or (c <= 0).any() or (d <= 0).any():
            return np.inf
        return nlp.f(z) - mu * (np.log(a[hasL]).sum() + np.log(b_[hasU]).sum()
                                + np.log(c[sHasL]).sum() + np.log(d[sHasU]).sum())

    def errors(z, s, yE, zLm, zUm, vL, vU, mu_t):
        yI = vU - vL
        JE = nlp.JE(z); JI = nlp.JI(z)
        rz = nlp.grad(z) + JE.T @ yE + JI.T @ yI - zLm + zUm
        cE = nlp.cE(z); cI = nlp.g(z) - s
        a, b_, c, d = gaps(z, s)
        comp = np.concatenate([(a * zLm - mu_t)[hasL], (b_ * zUm - mu_t)[hasU],
                               (c * vL - mu_t)[sHasL], (d * vU - mu_t)[sHasU]])
        ysum = np.abs(yE).sum() + np.abs(yI).sum()
        zsum = zLm.sum() + zUm.sum() + vL.sum() + vU.sum()
        sd = max(o.s_max, (ysum + zsum) / max(n_mult, 1)) / o.s_max
        sc = max(o.s_max, zsum / max(n_bmult, 1)) / o.s_max
        if o.dual_sum_groups:
            rz = rz.copy()
            tied = [rz[g].sum() for g in o.dual_sum_groups]
            for g in o.dual_sum_groups:
                rz[g] = 0.0
            rz = np.concatenate([rz, tied])
        dinf = np.abs(rz).max() if n else 0.0
        cinf = max(np.abs(cE).max() if mE else 0.0, np.abs(cI).max() if mI else 0.0)
        pinf = np.abs(comp).max() if comp.size else 0.0
        return max(dinf / sd, cinf, pinf / sc), dinf, cinf, pinf

    filt = []           # list of (theta, phi)
    n_kick = 0
    th0 = theta(z, s)
    theta_max = 1e4 * max(1.0, th0); theta_min = 1e-4 * max(1.0, th0)
    dw_last = 0.0
    log = []
    snaps = {}
    status = 0
    err = np.inf
    it = 0
    for it in range(o.max_iter + 1):
        if it in o.snapshots:
            snaps[it] = z.copy()
        e0, dinf, cinf, pinf = errors(z, s, yE, zLm, zUm, vL, vU, 0.0)
        err = e0
        if o.verbose:
            print(f"it {it:3d} f={nlp.f(z):.6e} th={theta(z, s):.2e} e0={e0:.2e} "
                  f"(d {dinf:.1e} c {cinf:.1e} p {pinf:.1e}) mu={mu:.1e} dw={dw_last:.1e}")
        if e0 <= o.tol and dinf <= o.dual_inf_tol and cinf <= o.constr_viol_tol and pinf <= o.compl_inf_tol:
            status = 1
            break
        if it == o.max_iter:
            status = 0
            break
        # ---- barrier parameter update (monotone) ----
        changed = False
        while mu > mu_min:
            emu = errors(z, s, yE, zLm, zUm, vL, vU, mu)[0]
            if emu > o.kappa_eps * mu:
                break
            mu = max(mu_min, min(o.kappa_mu * mu, mu ** o.theta_mu))
            tau = max(o.tau_min, 1 - mu)
            changed = True
        if changed:
            filt = []
        # ---- assemble condensed KKT ----
        yI = vU - vL
        a, b_, c, d = gaps(z, s)
        Sz = np.where(hasL, zLm / a, 0.0) + np.where(hasU, zUm / b_, 0.0)
        Ss = np.where(sHasL, vL / c, 0.0) + np.where(sHasU, vU / d, 0.0)
        W = nlp.hess(z, yE, yI)
        JE = nlp.JE(z); JI = nlp.JI(z)
        cE = nlp.cE(z); cI = nlp.g(z) - s
        gf = nlp.grad(z)
        bz = gf - np.where(hasL, mu / a, 0.0) + np.where(hasU, mu / b_, 0.0)
        gam = -np.where(sHasL, mu / c, 0.0) + np.where(sHasU, mu / d, 0.0)
        H0s = (W + sps.diags(Sz) + JI.T @ sps.diags(Ss) @ JI).tocsc()
        cE_eff = cE
        if o.freeze_degenerate > 0 and o.dc_rows is not None:
            rown = np.asarray(abs(JE).max(axis=1).todense()).ravel()
            frozen = (dc > 0) & (rown < o.freeze_degenerate)
            if frozen.any():
                cE_eff = np.where(frozen, 0.0, cE)
        rhs = np.concatenate([-(bz + JI.T @ (gam + Ss * cI)), -cE_eff - dc * yE])
        use_sparse = o.linsolve == "sparse"
        if not use_sparse:
            H0 = H0s.toarray(); JEd = JE.toarray()
        # ---- inertia correction (Algorithm IC) ----
        dw = 0.0
        ok = False
        first = True
        fac = None
        while True:
            sol = None
            if use_sparse:
                Ks = sps.bmat([[H0s + dw * sps.identity(n), JE.T], [JE, -sps.diags(dc + 0.0)]], format="csc")
                fac = _SparseLDL(Ks, o.order)
                if fac.ok and fac.npos == n and fac.nneg == mE and fac.nzero == 0:
                    sol = fac.solve(rhs)
                    if fac.resid < 1e-9:
                        ok = True
                        break
                    sol = None
                if not fac.ok or sol is None and fac.npos == n and fac.nneg == mE:
                    # SuperLU pivoted off the diagonal or lost accuracy: decide with the dense Bunch-Kaufman path
                    H0 = H0s.toarray(); JEd = JE.toarray()
                    use_dense_now = True
                else:
                    use_dense_now = False
            else:
                use_dense_now = True
            if use_dense_now:
                K = np.zeros((n + mE, n + mE))
                K[:n, :n] = H0 + dw * np.eye(n)
                K[n:, :n] = JEd
                K[n:, n:] = -np.diag(dc)
                ldu, ipiv, npos, nneg, nzero = _ldl_inertia(K)
                if npos == n and nneg == mE and nzero == 0:
                    ok = True
                    break
            if first:
                dw = o.dw_first if dw_last == 0.0 else max(o.dw_min, o.kw_minus * dw_last)
                first = False
            else:
                dw = dw * (o.kw_plus_first if dw_last == 0.0 else o.kw_plus)
            if dw > o.dw_max:
                break
        if not ok:
            status = -2
            break
        if dw > 0:
            dw_last = dw
        if sol is None:
            sol, info = lapack.dsytrs(ldu, ipiv, rhs, lower=1)
            # one step of iterative refinement
            Kfull = np.tril(K) + np.tril(K, -1).T
            res = rhs - Kfull @ sol
            sol = sol + lapack.dsytrs(ldu, ipiv, res, lower=1)[0]
        dz = sol[:n]; yEn = sol[n:]
        ds = JI @ dz + cI
        dzL = np.where(hasL, mu / a - zLm - zLm / a * dz, 0.0)
        dzU = np.where(hasU, mu / b_ - zUm + zUm / b_ * dz, 0.0)
        dvL = np.where(sHasL, mu / c - vL - vL / c * ds, 0.0)
        dvU = np.where(sHasU, mu / d - vU + vU / d * ds, 0.0)

        # ---- fraction to the boundary ----
        def amax(x, dx, mask):
            m = mask & (dx < 0)
            return min(1.0, (-tau * x[m] / dx[m]).min()) if m.any() else 1.0
        a_pr = min(amax(a, dz, hasL), amax(b_, -dz, hasU), amax(c, ds, sHasL), amax(d, -ds, sHasU))
        a_du = min(amax(zLm, dzL, hasL), amax(zUm, dzU, hasU), amax(vL, dvL, sHasL), amax(vU, dvU, sHasU))

        # ---- filter line search ----
        th_k = theta(z, s); ph_k = phi(z, s, mu)
        dphi = bz @ dz + gam @ ds
        if dphi < 0 and th_k <= theta_min:
            a_min = o.gamma_alpha * min(o.gamma_theta, o.gamma_phi * th_k / (-dphi),
                                        o.delta * th_k ** o.s_theta / (-dphi) ** o.s_phi)
        elif dphi < 0:
            a_min = o.gamma_alpha * min(o.gamma_theta, o.gamma_phi * th_k / (-dphi))
        else:
            a_min = o.gamma_alpha * o.gamma_theta
        alpha = a_pr
        accepted = False
        ftype = False
        nbt = 0
        while alpha >= a_min and nbt < o.max_backtrack:
            zt = z + alpha * dz; st = s + alpha * ds
            th_t = theta(zt, st); ph_t = phi(zt, st, mu)
            in_filter = th_t >= theta_max or any(th_t >= tf and ph_t >= pf for tf, pf in filt)
            if not in_filter and np.isfinite(ph_t):
                sw = dphi < 0 and alpha * (-dphi) ** o.s_phi > o.delta * th_k ** o.s_theta
                if th_k <= theta_min and sw:
                    if ph_t <= ph_k + o.eta_phi * alpha * dphi + 10 * np.finfo(float).eps * abs(ph_k):
                        accepted = True; ftype = True
                else:
                    if th_t <= (1 - o.gamma_theta) * th_k or ph_t <= ph_k - o.gamma_phi * th_k:
                        accepted = True
            if accepted:
                break
            alpha *= 0.5
            nbt += 1
        if not accepted:
            if n_kick < o.max_kick:             # "barrier kick" (restoration substitute, same rule as the CUDA solver)
                n_kick += 1
                filt = []
                mu = min(o.mu_init, 10.0 * mu)
                tau = max(o.tau_min, 1 - mu)
                continue
            status = -1
            break
        if not ftype:
            filt.append(((1 - o.gamma_theta) * th_k, ph_k - o.gamma_phi * th_k))
        # ---- accept ----
        a_y = min(alpha, a_du)          # alpha_for_y = "min"
        z = z + alpha * dz; s = s + alpha * ds
        yE = yE + a_y * (yEn - yE)
        zLm = zLm + a_du * dzL; zUm = zUm + a_du * dzU
        vL = vL + a_du * dvL; vU = vU + a_du * dvU
        a, b_, c, d = gaps(z, s)
        ks = o.kappa_sigma
        zLm = np.where(hasL, np.clip(zLm, mu / (ks * a), ks * mu / a), 0.0)
        zUm = np.where(hasU, np.clip(zUm, mu / (ks * b_), ks * mu / b_), 0.0)
        vL = np.where(sHasL, np.clip(vL, mu / (ks * c), ks * mu / c), 0.0)
        vU = np.where(sHasU, np.clip(vU, mu / (ks * d), ks * mu / d), 0.0)
        log.append(dict(it=it, mu=mu, alpha=alpha, a_du=a_du, dw=dw, nbt=nbt, th=th_k, e0=e0))
    return IpmResult(z, s, yE, vL, vU, zLm, zUm, status, it, err, mu, log, snaps)
