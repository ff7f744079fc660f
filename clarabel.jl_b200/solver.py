"""Interior-point driver: the *caller* of the KKT path.

Mirror of src/solver.jl (setup! :75-153, solve! :189-380, default start :383-404, strategy
checkpoints :453-514), src/variables.jl, src/residuals.jl, src/info.jl and src/solution.jl,
for symmetric cones (Zero/NN/SOC/PSD: every BASELINE config) and for the nonsymmetric ones
(exponential / power / generalised power: unit initialisation, primal-dual vs dual scaling
strategy with the reference's strategy checkpoints, barrier-limited steps).
It exists because "identical status codes / objectives" can only be judged through whole
solves and the reference's Julia loop cannot run here.  The loop is backend-agnostic: the
KKT solver is whatever `settings.direct_solve_method` names (kktsystem.py registry).

Timer sections use the reference's TimerOutputs names ("scale cones", "kkt update",
"kkt solve") because those are the numerator of the headline metric (BASELINE.md section 3).
"""
import time
import numpy as np
import scipy.sparse as sp

from .settings import Settings
from .cones import CompositeCone
from .problemdata import ProblemData
from .kktsystem import DefaultKKTSystem
from .nonsymmetric import PRIMAL_DUAL, DUAL

# statuscodes.jl:24-36
(UNSOLVED, SOLVED, PRIMAL_INFEASIBLE, DUAL_INFEASIBLE, ALMOST_SOLVED,
 ALMOST_PRIMAL_INFEASIBLE, ALMOST_DUAL_INFEASIBLE, MAX_ITERATIONS, MAX_TIME,
 NUMERICAL_ERROR, INSUFFICIENT_PROGRESS) = range(11)
STATUS_NAMES = ["UNSOLVED", "SOLVED", "PRIMAL_INFEASIBLE", "DUAL_INFEASIBLE", "ALMOST_SOLVED",
                "ALMOST_PRIMAL_INFEASIBLE", "ALMOST_DUAL_INFEASIBLE", "MAX_ITERATIONS",
                "MAX_TIME", "NUMERICAL_ERROR", "INSUFFICIENT_PROGRESS"]
_EPS = float(np.finfo(np.float64).eps)
_FLOATMAX = float(np.finfo(np.float64).max)


class Variables:
    def __init__(self, n, m):
        self.x = np.zeros(n); self.s = np.zeros(m); self.z = np.zeros(m)
        self.tau = 1.0; self.kappa = 1.0

    def copy_from(self, o):
        self.x[:] = o.x; self.s[:] = o.s; self.z[:] = o.z
        self.tau = o.tau; self.kappa = o.kappa


class Residuals:
    def __init__(self, n, m):
        self.rx = np.zeros(n); self.rz = np.zeros(m); self.rtau = 1.0
        self.rx_inf = np.zeros(n); self.rz_inf = np.zeros(m); self.Px = np.zeros(n)
        self.dot_qx = self.dot_bz = self.dot_sz = self.dot_xPx = 0.0

    def update(self, v, data):
        """residuals_update! (residuals.jl:1-37)."""
        P, A = data.P, data.A
        qx = float(data.q @ v.x); bz = float(data.b @ v.z); sz = float(v.s @ v.z)
        if P.nnz:
            self.Px[:] = P @ v.x + P.T @ v.x - P.diagonal() * v.x
        else:
            self.Px[:] = 0.0
        xPx = float(v.x @ self.Px)
        self.rx_inf[:] = -(A.T @ v.z)
        self.rz_inf[:] = v.s + A @ v.x
        self.rx[:] = self.rx_inf - self.Px - data.q * v.tau
        self.rz[:] = self.rz_inf - data.b * v.tau
        self.rtau = qx + bz + v.kappa + xPx / v.tau
        self.dot_qx, self.dot_bz, self.dot_sz, self.dot_xPx = qx, bz, sz, xPx


class Info:
    def __init__(self):
        self.status = UNSOLVED
        self.iterations = 0
        self.mu = self.sigma = self.step_length = 0.0
        self.cost_primal = self.cost_dual = 0.0
        self.res_primal = self.res_dual = 0.0
        self.res_primal_inf = self.res_dual_inf = 0.0
        self.gap_abs = self.gap_rel = 0.0
        self.ktratio = 0.0
        self.prev_cost_primal = self.prev_cost_dual = 0.0
        self.prev_res_primal = self.prev_res_dual = 0.0
        self.prev_gap_abs = self.prev_gap_rel = 0.0
        self.solve_time = 0.0
        self.linsolver = None


def _norm_scaled(x, v):
    return float(np.linalg.norm(x * v))


class Solution:
    pass


class Solver:
    def __init__(self, P, q, A, b, cones, settings=None):
        self.settings = settings if settings is not None else Settings()
        self.timers = {"setup!": 0.0, "equilibration": 0.0, "kkt init": 0.0, "solve!": 0.0,
                       "default start": 0.0, "scale cones": 0.0, "kkt update": 0.0,
                       "kkt solve": 0.0}
        t0 = time.perf_counter()
        st = self.settings
        self.info = Info()
        self.data = ProblemData(P, q, A, b, cones, st)
        self.cones = CompositeCone(self.data.cones)
        if self.data.m != self.cones.numel:
            raise ValueError("Constraint dimensions inconsistent with size of cones.")
        n, m = self.data.n, self.data.m
        if len(self.data.q) != n or self.data.P.shape != (n, n) or len(self.data.b) != m:
            raise ValueError("problem dimension mismatch")
        self.variables = Variables(n, m)
        self.residuals = Residuals(n, m)
        t1 = time.perf_counter()
        self.data.equilibrate(self.cones, st)
        self.timers["equilibration"] = time.perf_counter() - t1
        t1 = time.perf_counter()
        self.kktsystem = DefaultKKTSystem(self.data, self.cones, st)
        self.timers["kkt init"] = time.perf_counter() - t1
        self.info.linsolver = self.kktsystem.linear_solver_info()
        self.step_rhs = Variables(n, m)
        self.step_lhs = Variables(n, m)
        self.prev_vars = Variables(n, m)
        self.solution = Solution()
        self.timers["setup!"] = time.perf_counter() - t0

    # ------------------------------------------------------------- fixtures
    def save_to_file(self, path):
        """save_to_file (src/json.jl:24-54): the problem as the solver holds it (after presolve),
        in unscaled form, in the reference's JSON schema."""
        import dataclasses
        from .problems import to_reference_json
        d = self.data
        P = d.P.copy(); A = d.A.copy()
        Pc = np.repeat(np.arange(d.n), np.diff(P.indptr)); Ac = np.repeat(np.arange(d.n), np.diff(A.indptr))
        P.data *= d.dinv[P.indices] * d.dinv[Pc] / d.c
        A.data *= d.einv[A.indices] * d.dinv[Ac]
        st = {}
        for k, v in dataclasses.asdict(self.settings).items():
            if isinstance(v, float) and np.isinf(v):
                v = float(np.sign(v) * np.finfo(np.float64).max)       # sanitize_settings!
            st[k] = v
        to_reference_json(path, P, d.q * d.dinv / d.c, A, d.b * d.einv, d.cones, st)

    @classmethod
    def load_from_file(cls, path, settings=None):
        """load_from_file (src/json.jl:58-80); `settings` overrides the stored ones."""
        from .problems import from_reference_json
        P, q, A, b, cones, st = from_reference_json(path)
        if settings is None:
            settings = Settings()
            fmax = float(np.finfo(np.float64).max)
            for k, v in st.items():
                if hasattr(settings, k):
                    if isinstance(v, float) and abs(v) == fmax:
                        v = float(np.sign(v) * np.inf)                  # desanitize_settings!
                    setattr(settings, k, type(getattr(settings, k))(v))
        return cls(P, q, A, b, cones, settings)

    # ---------------------------------------------------------- data updates
    # src/data_updating.jl:22-160: overwrite P / q / A / b in place (same sparsity pattern), scaled
    # with the equilibration computed at setup, and push the new values to the KKT solver through
    # kktsolver_update_P!/A! (no new symbolic analysis).  `data` may be None (no-op), a vector of
    # the stored nonzeros / entries, a scipy matrix with the stored pattern, or an iterable of
    # (index, value) pairs with 0-based indices into the stored values.
    def _check_data_update_allowed(self):
        if self.data.presolve_keep is not None:
            raise RuntimeError("Data updates not allowed if presolver is active.")
        if self.data.dropped_zeros:
            raise RuntimeError("Data updates not allowed if sparse zeros are dropped.")

    @staticmethod
    def _pairs(data):
        """list of (index, value) pairs if `data` is the zip / pair-sequence form, else None"""
        if sp.issparse(data) or isinstance(data, np.ndarray):
            return None
        if hasattr(data, "__len__"):
            seq = list(data)
            if seq and isinstance(seq[0], (tuple, list)) and len(seq[0]) == 2:
                return seq
            return None
        return list(data)

    def _update_matrix(self, data, M, lscale, rscale, cscale):
        if sp.issparse(data):
            D = sp.csc_matrix(data, dtype=np.float64); D.sort_indices()
            if (D.shape != M.shape or not np.array_equal(D.indptr, M.indptr)
                    or not np.array_equal(D.indices, M.indices)):
                raise ValueError("Input must match sparsity pattern of original data.")
            data = D.data
        cols = np.repeat(np.arange(M.shape[1]), np.diff(M.indptr))
        pairs = self._pairs(data)
        if pairs is not None:
            for idx, value in pairs:
                if not 0 <= idx < M.nnz:
                    raise ValueError("Input must match sparsity pattern of original data.")
                v = lscale[M.indices[idx]] * rscale[cols[idx]] * value
                M.data[idx] = v if cscale is None else v * cscale
            return True
        data = np.asarray(data, dtype=np.float64)
        if len(data) == 0:
            return False
        if len(data) != M.nnz:
            raise ValueError("Input must match length of original data.")
        M.data[:] = data * lscale[M.indices] * rscale[cols]
        if cscale is not None:
            M.data *= cscale
        return True

    @staticmethod
    def _update_vector(data, v, vscale, cscale):
        c = 1.0 if cscale is None else cscale
        pairs = Solver._pairs(data)
        if pairs is not None:
            for idx, value in pairs:
                v[idx] = value * vscale[idx] * c
            return True
        data = np.asarray(data, dtype=np.float64)
        if len(data) == 0:
            return False
        if len(data) != len(v):
            raise ValueError("Input must match length of original data.")
        v[:] = data * vscale * c
        return True

    def update_P(self, data):
        """update_P! (data_updating.jl:56-69); a matrix argument is the upper triangle of P."""
        if data is None:
            return
        self._check_data_update_allowed()
        d = self.data.d
        if self._update_matrix(data, self.data.P, d, d, self.data.c):
            self.kktsystem.update_P(self.data.P)

    def update_A(self, data):
        """update_A! (data_updating.jl:86-99)."""
        if data is None:
            return
        self._check_data_update_allowed()
        if self._update_matrix(data, self.data.A, self.data.e, self.data.d, None):
            self.kktsystem.update_A(self.data.A)

    def update_q(self, data):
        """update_q! (data_updating.jl:108-122)."""
        if data is None:
            return
        self._check_data_update_allowed()
        if self._update_vector(data, self.data.q, self.data.d, self.data.c):
            self.data.normq = None

    def update_b(self, data):
        """update_b! (data_updating.jl:131-144)."""
        if data is None:
            return
        self._check_data_update_allowed()
        if self._update_vector(data, self.data.b, self.data.e, None):
            self.data.normb = None

    def update_data(self, P=None, q=None, A=None, b=None):
        """update_data! (data_updating.jl:22-37)."""
        self.update_P(P); self.update_q(q); self.update_A(A); self.update_b(b)

    # ------------------------------------------------------------------ info
    def _info_update(self):
        """info_update! (info.jl:1-63)."""
        info, data, v, r = self.info, self.data, self.variables, self.residuals
        tauinv = 1.0 / v.tau
        normb, normq = data.get_normb(), data.get_normq()
        d, dinv, e, einv = data.d, data.dinv, data.e, data.einv
        cinv = 1.0 / data.c
        xPx_t = r.dot_xPx * tauinv * tauinv / 2
        info.cost_primal = (r.dot_qx * tauinv + xPx_t) * cinv
        info.cost_dual = (-r.dot_bz * tauinv - xPx_t) * cinv
        normx = _norm_scaled(d, v.x)
        normz = _norm_scaled(e, v.z) * cinv
        norms = _norm_scaled(einv, v.s)
        info.res_primal_inf = (_norm_scaled(dinv, r.rx_inf) * cinv) / max(1.0, normz)
        info.res_dual_inf = max(_norm_scaled(dinv, r.Px) / max(1.0, normx),
                                _norm_scaled(einv, r.rz_inf) / max(1.0, normx + norms))
        normx *= tauinv; normz *= tauinv; norms *= tauinv
        info.res_primal = _norm_scaled(einv, r.rz) * tauinv / max(1.0, normb + normx + norms)
        info.res_dual = _norm_scaled(dinv, r.rx) * tauinv * cinv / max(1.0, normq + normx + normz)
        info.gap_abs = abs(info.cost_primal - info.cost_dual)
        info.gap_rel = info.gap_abs / max(1.0, min(abs(info.cost_primal), abs(info.cost_dual)))
        info.ktratio = v.kappa * tauinv
        info.solve_time = time.perf_counter() - self._t_solve0

    def _check_convergence(self, full):
        info, r, st = self.info, self.residuals, self.settings
        if full:
            tg_a, tg_r, tf = st.tol_gap_abs, st.tol_gap_rel, st.tol_feas
            ti_a, ti_r, tk = st.tol_infeas_abs, st.tol_infeas_rel, st.tol_ktratio
            s_ok, s_p, s_d = SOLVED, PRIMAL_INFEASIBLE, DUAL_INFEASIBLE
        else:
            tg_a, tg_r, tf = st.reduced_tol_gap_abs, st.reduced_tol_gap_rel, st.reduced_tol_feas
            ti_a, ti_r, tk = (st.reduced_tol_infeas_abs, st.reduced_tol_infeas_rel,
                              st.reduced_tol_ktratio)
            s_ok, s_p, s_d = ALMOST_SOLVED, ALMOST_PRIMAL_INFEASIBLE, ALMOST_DUAL_INFEASIBLE
        is_solved = (((info.gap_abs < tg_a) or (info.gap_rel < tg_r))
                     and info.res_primal < tf and info.res_dual < tf)
        if info.ktratio <= 1.0 and is_solved:
            info.status = s_ok
        elif info.ktratio > 1000.0 / tk:
            if (r.dot_bz < -ti_a) and (info.res_primal_inf < -ti_r * r.dot_bz):
                info.status = s_p
            elif (r.dot_qx < -ti_a) and (info.res_dual_inf < -ti_r * r.dot_qx):
                info.status = s_d

    def _check_termination(self, it):
        """info_check_termination! (info.jl:65-120)."""
        info, st = self.info, self.settings
        info.status = UNSOLVED
        self._check_convergence(True)
        if (info.status == UNSOLVED and it > 1 and
                (info.res_dual > info.prev_res_dual or info.res_primal > info.prev_res_primal)):
            if info.ktratio < 100 * _EPS and (info.prev_gap_abs < st.tol_gap_abs or
                                               info.prev_gap_rel < st.tol_gap_rel):
                info.status = INSUFFICIENT_PROGRESS
            if info.ktratio < 1.0:
                if ((info.res_dual > 100 * st.tol_feas and info.res_dual > 100 * info.prev_res_dual) or
                        (info.res_primal > 100 * st.tol_feas and info.res_primal > 100 * info.prev_res_primal)):
                    info.status = INSUFFICIENT_PROGRESS
        if info.status == UNSOLVED:
            if st.max_iter == info.iterations:
                info.status = MAX_ITERATIONS
            elif info.solve_time > st.time_limit:
                info.status = MAX_TIME
        return info.status != UNSOLVED

    def _save_prev(self):
        i = self.info
        i.prev_cost_primal, i.prev_cost_dual = i.cost_primal, i.cost_dual
        i.prev_res_primal, i.prev_res_dual = i.res_primal, i.res_dual
        i.prev_gap_abs, i.prev_gap_rel = i.gap_abs, i.gap_rel
        self.prev_vars.copy_from(self.variables)

    def _reset_to_prev(self):
        i = self.info
        i.cost_primal, i.cost_dual = i.prev_cost_primal, i.prev_cost_dual
        i.res_primal, i.res_dual = i.prev_res_primal, i.prev_res_dual
        i.gap_abs, i.gap_rel = i.prev_gap_abs, i.prev_gap_rel
        self.variables.copy_from(self.prev_vars)

    # ------------------------------------------------------------- variables
    def _calc_step_length(self, steptype, scaling=PRIMAL_DUAL):
        """solver_get_step_length (solver.jl:407-422) = variables_calc_step_length
        (variables.jl:14-46) + the barrier limit for nonsymmetric cones under dual scaling."""
        v, step = self.variables, self.step_lhs
        a_tau = -v.tau / step.tau if step.tau < 0 else _FLOATMAX
        a_kap = -v.kappa / step.kappa if step.kappa < 0 else _FLOATMAX
        a = min(a_tau, a_kap, 1.0)
        az, as_ = self.cones.step_length(step.z, step.s, v.z, v.s, a, self.settings)
        a = min(az, as_)
        if steptype == "combined":
            a *= self.settings.max_step_fraction
        if (not self.cones.is_symmetric) and steptype == "combined" and scaling == DUAL:
            a = self._backtrack_step_to_barrier(a)
        return a

    def _barrier(self, a):
        """variables_barrier (variables.jl:46-72)."""
        v, step, cones = self.variables, self.step_lhs, self.cones
        coef = cones.degree + 1
        tau, kap = v.tau + a * step.tau, v.kappa + a * step.kappa
        sz = float((v.z + a * step.z) @ (v.s + a * step.s))
        mu = (sz + tau * kap) / coef
        if mu <= 0 or tau <= 0 or kap <= 0:
            return np.inf
        return (coef * np.log(mu) - np.log(tau) - np.log(kap)
                + cones.compute_barrier(v.z, v.s, step.z, step.s, a))

    def _backtrack_step_to_barrier(self, a):
        """solver_backtrack_step_to_barrier (solver.jl:425-442)."""
        back = self.settings.linesearch_backtrack_step
        for _ in range(50):
            if self._barrier(a) < 1.0:
                return a
            a *= back
        return a

    def _shift_to_cone_interior(self, z, pd):
        """_shift_to_cone_interior! (variables.jl:176-206)."""
        cones = self.cones
        min_margin, pos_margin = cones.margins(z, pd)
        target = max(1.0, 0.1 * pos_margin / cones.degree) if cones.degree > 0 else 1.0
        if min_margin <= 0:
            cones.scaled_unit_shift(z, -min_margin, pd)
            cones.scaled_unit_shift(z, target, pd)
        elif min_margin < target:
            cones.scaled_unit_shift(z, target - min_margin, pd)
        else:
            cones.scaled_unit_shift(z, 0.0, pd)

    def _default_start(self):
        """solver_default_start! (solver.jl:383-404)."""
        if not self.cones.is_symmetric:
            # variables_unit_initialization! (variables.jl:213-226)
            v = self.variables
            self.cones.unit_initialization(v.z, v.s)
            v.x[:] = 0.0; v.tau = 1.0; v.kappa = 1.0
            return
        self.cones.set_identity_scaling()
        self.kktsystem.update(self.data, self.cones)
        self.kktsystem.solve_initial_point(self.variables, self.data)
        self._shift_to_cone_interior(self.variables.s, "primal")
        self._shift_to_cone_interior(self.variables.z, "dual")
        self.variables.tau = 1.0
        self.variables.kappa = 1.0

    # ------------------------------------------------------------------ solve
    def solve(self, max_iter=None):
        st = self.settings
        if max_iter is not None:
            st.max_iter = max_iter
        info, data, cones = self.info, self.data, self.cones
        v, r = self.variables, self.residuals
        tm = self.timers
        for k in ("scale cones", "kkt update", "kkt solve", "default start", "solve!"):
            tm[k] = 0.0
        it = 0
        sigma, alpha, mu = 1.0, 0.0, _FLOATMAX
        info.status = UNSOLVED; info.iterations = 0
        self._t_solve0 = time.perf_counter()
        t = time.perf_counter()
        self._default_start()
        tm["default start"] = time.perf_counter() - t
        self.iter_log = []
        sym = cones.is_symmetric
        scaling = PRIMAL_DUAL if cones.allows_primal_dual_scaling else DUAL
        # NT scaling of the symmetric cones on the device (the state stays there for the next kkt update)
        device_scaling = st.b200_device_cone_scaling and st.direct_solve_method == "b200" and sym
        while True:
            r.update(v, data)
            mu = (r.dot_sz + v.tau * v.kappa) / (cones.degree + 1)
            info.mu, info.step_length, info.sigma, info.iterations = mu, alpha, sigma, it
            self._info_update()
            self.iter_log.append((it, info.cost_primal, info.cost_dual, info.res_primal,
                                  info.res_dual, mu, alpha))
            if st.verbose:
                print(f"{it:3d} pcost {info.cost_primal: .6e} dcost {info.cost_dual: .6e} "
                      f"gap {info.gap_abs:.2e} pres {info.res_primal:.2e} dres {info.res_dual:.2e} "
                      f"k/t {info.ktratio:.2e} mu {mu:.2e} step {alpha:.2e}")
            if self._check_termination(it):
                # _strategy_checkpoint_insufficient_progress (solver.jl:453-472)
                if info.status == INSUFFICIENT_PROGRESS:
                    self._reset_to_prev()
                    if (not sym) and scaling == PRIMAL_DUAL:
                        info.status = UNSOLVED
                        scaling = DUAL
                        continue
                break
            t = time.perf_counter()
            if device_scaling:
                ok_scale = self.kktsystem.kktsolver.update_scaling(v.s, v.z, cones)
            else:
                ok_scale = cones.update_scaling(v.s, v.z, mu, scaling)
            tm["scale cones"] += time.perf_counter() - t
            if not ok_scale:
                info.status = NUMERICAL_ERROR
                break
            it += 1
            t = time.perf_counter()
            ok = self.kktsystem.update(data, cones)
            tm["kkt update"] += time.perf_counter() - t
            # affine step rhs (variables.jl:107-122)
            d = self.step_rhs
            d.x[:] = r.rx; d.z[:] = r.rz
            cones.affine_ds(d.s, v.s)
            d.tau = r.rtau; d.kappa = v.tau * v.kappa
            if ok:
                t = time.perf_counter()
                ok = self.kktsystem.solve(self.step_lhs, d, data, v, cones, "affine")
                tm["kkt solve"] += time.perf_counter() - t
            if ok:
                alpha = self._calc_step_length("affine", scaling)
                sigma = (1.0 - alpha) ** 3
                mm = 1.0 if it > 1 else alpha
                # combined step rhs (variables.jl:125-168)
                step = self.step_lhs
                sm = sigma * mu
                d.x[:] = (1.0 - sigma) * r.rx
                d.tau = (1.0 - sigma) * r.rtau
                d.kappa = -sm + mm * step.tau * step.kappa + v.tau * v.kappa
                if mm != 1.0:
                    step.z *= mm
                cones.combined_ds_shift(d.z, step.z, step.s, sm)
                d.s += d.z
                d.z[:] = (1.0 - sigma) * r.rz
                t = time.perf_counter()
                ok = self.kktsystem.solve(self.step_lhs, d, data, v, cones, "combined")
                tm["kkt solve"] += time.perf_counter() - t
            if not ok:
                # _strategy_checkpoint_numerical_error (solver.jl:475-489)
                alpha = 0.0
                if (not sym) and scaling == PRIMAL_DUAL:
                    scaling = DUAL
                    continue
                info.status = NUMERICAL_ERROR
                break
            alpha = self._calc_step_length("combined", scaling)
            # _strategy_checkpoint_small_step (solver.jl:492-505)
            if (not sym) and scaling == PRIMAL_DUAL and alpha < st.min_switch_step_length:
                scaling = DUAL
                alpha = 0.0
                continue
            if alpha <= max(0.0, st.min_terminate_step_length):
                info.status = INSUFFICIENT_PROGRESS
                alpha = 0.0
                break
            self._save_prev()
            v.x += alpha * self.step_lhs.x
            v.s += alpha * self.step_lhs.s
            v.z += alpha * self.step_lhs.z
            v.tau += alpha * self.step_lhs.tau
            v.kappa += alpha * self.step_lhs.kappa
        tm["solve!"] = time.perf_counter() - self._t_solve0
        if alpha == 0.0:
            info.mu, info.step_length, info.sigma, info.iterations = mu, alpha, sigma, it
        # post-process (info.jl:196-213, solution.jl:2-50)
        if info.status in (NUMERICAL_ERROR, INSUFFICIENT_PROGRESS, MAX_ITERATIONS, MAX_TIME):
            self._check_convergence(False)
        sol = self.solution
        sol.status = info.status
        infeas = info.status in (PRIMAL_INFEASIBLE, DUAL_INFEASIBLE,
                                 ALMOST_PRIMAL_INFEASIBLE, ALMOST_DUAL_INFEASIBLE)
        sol.obj_val = float("nan") if infeas else info.cost_primal
        sol.obj_val_dual = float("nan") if infeas else info.cost_dual
        sol.iterations = info.iterations
        sol.r_prim, sol.r_dual = info.res_primal, info.res_dual
        scaleinv = 1.0 / (v.kappa if infeas else v.tau)
        cinv = 1.0 / data.c
        sol.x = v.x * data.d * scaleinv
        sol.z = v.z * data.e * (scaleinv * cinv)
        sol.s = v.s * data.einv * scaleinv
        if data.presolve_keep is not None:
            # reverse_presolve! (presolver.jl:82-104): removed rows get s = infinity, z = 0
            from .problemdata import INFINITY
            keep = data.presolve_keep
            zf = np.zeros(data.mfull); sf = np.full(data.mfull, INFINITY)
            zf[keep] = sol.z; sf[keep] = sol.s
            sol.z, sol.s = zf, sf
        info.solve_time = time.perf_counter() - self._t_solve0
        sol.solve_time = info.solve_time
        sol.status_name = STATUS_NAMES[sol.status]
        return sol
