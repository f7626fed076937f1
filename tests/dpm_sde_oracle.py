"""Float64 restatement of the SDE variant of DPM-Solver++(2M) (Lu et al. 2022, "DPM-Solver++", the data-prediction SDE solver
in its second-order multistep midpoint form, as diffusers' "sde-dpmsolver++") with injected noise, and the exact first two
moments of a linear solver's output on Gaussian data.

Test infrastructure next to tests/dpm_oracle.py (the ODE solver), which it reuses and leaves as it is.  The product's path is
DPMSolverSchedule(sde=True) (coefficient rows) + k2_dpm_solver_sde_step (one row per step).
"""
import numpy as np

from tests import dpm_oracle as do


def solve_sde(eps_fn, x, alpha, sigma, noise, first=0, order=2, inpaint=None):
    """From x at grid point `first` to grid point n; noise[j] is the Gaussian draw of the j-th step run (k = first + j).
    Per step, with D_k = (x_k - sigma_k eps) / alpha_k and h_k = lambda_{k+1} - lambda_k:
        x_{k+1} = sigma_{k+1}/sigma_k e^{-h} x_k + alpha_{k+1} (1 - e^{-2h}) D' + sigma_{k+1} sqrt(1 - e^{-2h}) z_k,
        D' = D_k on first-order steps, else (1 + 1/(2r)) D_k - 1/(2r) D_{k-1} with r = h_{k-1} / h_k;
    a target sigma_{k+1} = 0 gives x_{k+1} = D_k.  inpaint = (init, mask, noise0) as in dpm_oracle.solve (Kandinsky 2.2).
    Works on numpy arrays and torch tensors alike."""
    n = len(alpha) - 1
    lam = [float(v) for v in do._lam(np.asarray(alpha), np.asarray(sigma))]
    alpha, sigma = [float(v) for v in alpha], [float(v) for v in sigma]
    d_prev, h_prev = None, None
    for k in range(first, n):
        d = (x - sigma[k] * eps_fn(x, k)) / alpha[k]
        if sigma[k + 1] == 0.0:
            x = d
        else:
            h = lam[k + 1] - lam[k]
            if order == 2 and d_prev is not None:
                r = h_prev / h
                dd = (1.0 + 1.0 / (2.0 * r)) * d - 1.0 / (2.0 * r) * d_prev
            else:
                dd = d
            one_m = -float(np.expm1(-2.0 * h))                 # 1 - e^{-2h}
            x = sigma[k + 1] / sigma[k] * float(np.exp(-h)) * x + alpha[k + 1] * one_m * dd + \
                sigma[k + 1] * one_m ** 0.5 * noise[k - first]
            h_prev = h
        d_prev = d
        if inpaint is not None:
            init, mask, noise0 = inpaint
            x = mask * (alpha[k + 1] * init + sigma[k + 1] * noise0) + (1 - mask) * x
    return x


def sde_rows(alpha, sigma, first=0, order=2):
    """Rows {1/a_k, s_k/a_k, c_x, c_D, c_P, a_{k+1}, s_{k+1}, c_N} of steps first .. n-1 (float64, step order) on any grid, the
    target sigma_n may be interior (the convergence tests).  order=1 drops the D_{k-1} term everywhere."""
    n = len(alpha) - 1
    lam = do._lam(alpha, sigma)
    out = []
    for k in range(first, n):
        row = np.zeros(8)
        row[0], row[1], row[5], row[6] = 1.0 / alpha[k], sigma[k] / alpha[k], alpha[k + 1], sigma[k + 1]
        if sigma[k + 1] == 0.0:
            row[3] = 1.0
        else:
            h = lam[k + 1] - lam[k]
            c = alpha[k + 1] * (1.0 - np.exp(-2.0 * h))
            row[2] = sigma[k + 1] / sigma[k] * np.exp(-h)
            row[7] = sigma[k + 1] * np.sqrt(1.0 - np.exp(-2.0 * h))
            if order == 1 or k == first:
                row[3] = c
            else:
                r = (lam[k] - lam[k - 1]) / h
                row[3], row[4] = c * (1.0 + 1.0 / (2.0 * r)), -c / (2.0 * r)
        out.append(row)
    return np.array(out).reshape(-1, 8)


def apply_rows_sde(table, eps_fn, x, noise, step_index=None):
    """The kernel's formula row by row in float64: x' = c_x x + c_D x0 + c_P hist + c_N z; hist read only when c_P != 0 and z
    only when c_N != 0."""
    hist = None
    for j, row in enumerate(table):
        k = j if step_index is None else step_index[j]
        x0 = row[0] * x - row[1] * eps_fn(x, k)
        xn = row[2] * x + row[3] * x0
        if row[4] != 0.0:
            xn = xn + row[4] * hist
        if row[7] != 0.0:
            xn = xn + row[7] * noise[j]
        hist, x = x0, xn
    return x


def gaussian_moments(table, alpha, sigma, mu, s):
    """Exact mean and variance of the output of the rows (applied with the kernel's formula, step k = row k) on Gaussian data
    x0 ~ N(mu, s^2), started from the exact marginal at grid point 0 and given the exact epsilon-predictor.  Every step is
    linear in the state (x_k, D_{k-1}, 1) plus independent noise c_N z, so its mean and covariance propagate in closed form."""
    m = np.array([alpha[0] * mu, 0.0, 1.0])
    P = np.zeros((3, 3))
    P[0, 0] = alpha[0] ** 2 * s ** 2 + sigma[0] ** 2
    for k, row in enumerate(table):
        den = alpha[k] ** 2 * s ** 2 + sigma[k] ** 2
        # D = (x - sigma eps) / alpha with eps = gaussian_eps: D = dA x + dB
        dA, dB = (1.0 - sigma[k] ** 2 / den) / alpha[k], sigma[k] ** 2 * mu / den
        cx, cD, cP, cN = row[2], row[3], row[4], row[7]
        M = np.array([[cx + cD * dA, cP, cD * dB], [dA, 0.0, dB], [0.0, 0.0, 1.0]])
        m = M @ m
        P = M @ P @ M.T
        P[0, 0] += cN ** 2
    return m[0], P[0, 0]
