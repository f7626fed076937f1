"""Float64 restatement of DPM-Solver++(2M) (Lu et al. 2022, "DPM-Solver++: Fast Solver for Guided Sampling of Diffusion
Probabilistic Models", Algorithm 2) and of a Gaussian-data problem whose probability-flow ODE has a closed form.

Test infrastructure.  It restates the paper, not the reference (which has no DPM solver), so it lives next to the tests like
tests/lora_oracle.py rather than in oracle/.  The product's path is kandinsky2/model/gaussian_diffusion.py: DPMSolverSchedule
(coefficient rows) + k2_dpm_solver_step (one row per step); here the update is written in the paper's form instead.
"""
import numpy as np


def timesteps(n, train_steps=1000):
    """tau_0 > ... > tau_{n-1}: the n evaluation timesteps ("linspace" spacing, the last grid point 0 dropped)."""
    return np.linspace(0, train_steps - 1, n + 1).round()[::-1][:n].astype(np.int64)


def grid(alphas_cumprod, n, train_steps=1000):
    """(tau [n], alpha [n+1], sigma [n+1]) of an n-step run: the evaluation points, then the target alpha = 1, sigma = 0."""
    tau = timesteps(n, train_steps)
    ac = np.asarray(alphas_cumprod, dtype=np.float64)[tau]
    return tau, np.append(np.sqrt(ac), 1.0), np.append(np.sqrt(1.0 - ac), 0.0)


def _lam(alpha, sigma):
    with np.errstate(divide="ignore"):
        return np.log(alpha) - np.log(sigma)


def rows(alpha, sigma, first=0, order=2):
    """Coefficient rows {1/a_k, s_k/a_k, c_x, c_D, c_P, a_{k+1}, s_{k+1}, 0} of steps k = first .. n-1 (float64, step order)
    on any grid alpha / sigma [n+1] -- the target sigma_n may be 0 (the sampler's) or interior (the convergence tests).
    x_{k+1} = c_x x_k + c_D D_k + c_P D_{k-1} restates Algorithm 2's
        x_{k+1} = sigma_{k+1}/sigma_k x_k - alpha_{k+1} (e^{-h_k} - 1) [(1 + 1/(2 r_k)) D_k - 1/(2 r_k) D_{k-1}].
    order=1 drops the D_{k-1} term everywhere (DPM-Solver++(1), i.e. DDIM in x0 form)."""
    n = len(alpha) - 1
    lam = _lam(alpha, sigma)
    out = []
    for k in range(first, n):
        row = np.zeros(8)
        row[0], row[1], row[5], row[6] = 1.0 / alpha[k], sigma[k] / alpha[k], alpha[k + 1], sigma[k + 1]
        if sigma[k + 1] == 0.0:          # h = inf: the step lands on D_k
            row[3] = 1.0
        else:
            h = lam[k + 1] - lam[k]
            c = alpha[k + 1] * (1.0 - np.exp(-h))
            row[2] = sigma[k + 1] / sigma[k]
            if order == 1 or k == first:
                row[3] = c
            else:
                r = (lam[k] - lam[k - 1]) / h
                row[3], row[4] = c * (1.0 + 1.0 / (2.0 * r)), -c / (2.0 * r)
        out.append(row)
    return np.array(out).reshape(-1, 8)


def solve(eps_fn, x, alpha, sigma, first=0, order=2, inpaint=None):
    """Algorithm 2 from x at grid point `first` to grid point n.  eps_fn(x, k) -> the (guided) epsilon at grid point k.
    inpaint = (init, mask, noise0): Kandinsky 2.2's rule -- after every step the known region (mask 1) is init noised to the
    next grid point with noise0.  Works on numpy arrays and torch tensors alike."""
    n = len(alpha) - 1
    lam = [float(v) for v in _lam(np.asarray(alpha), np.asarray(sigma))]
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
            x = sigma[k + 1] / sigma[k] * x - alpha[k + 1] * float(np.expm1(-h)) * dd
            h_prev = h
        d_prev = d
        if inpaint is not None:
            init, mask, noise0 = inpaint
            x = mask * (alpha[k + 1] * init + sigma[k + 1] * noise0) + (1 - mask) * x
    return x


def apply_rows(table, eps_fn, x, step_index=None):
    """The kernel's formula evaluated row by row in float64: x' = c_x x + c_D x0 + c_P hist, hist read only when c_P != 0."""
    hist = None
    for j, row in enumerate(table):
        k = j if step_index is None else step_index[j]
        x0 = row[0] * x - row[1] * eps_fn(x, k)
        xn = row[2] * x + row[3] * x0
        if row[4] != 0.0:
            xn = xn + row[4] * hist
        hist, x = x0, xn
    return x


# ---- Gaussian data: x0 ~ N(mu, s^2) elementwise ------------------------------------------------------------------------
def gaussian_eps(x, alpha, sigma, mu, s):
    """The exact epsilon-predictor E[eps | x_t = x] for x_t = alpha x0 + sigma eps."""
    return sigma * (x - alpha * mu) / (alpha ** 2 * s ** 2 + sigma ** 2)


def gaussian_flow(x, alpha_a, sigma_a, alpha_b, sigma_b, mu, s):
    """The probability-flow ODE's map from (alpha_a, sigma_a) to (alpha_b, sigma_b)."""
    return alpha_b * mu + np.sqrt(alpha_b ** 2 * s ** 2 + sigma_b ** 2) * (x - alpha_a * mu) / np.sqrt(
        alpha_a ** 2 * s ** 2 + sigma_a ** 2)


def smooth_grid(n, t_start=999.0, t_end=200.0, beta_start=0.00085, beta_end=0.012, train_steps=1000):
    """n steps uniform in continuous time from t_start to t_end (interior: sigma > 0 at both ends) of the continuous linear-beta
    schedule log abar(t) = -int_0^t beta, beta linear from beta_start to beta_end over [0, train_steps - 1].  Nested under
    doubling, so the error against gaussian_flow shows the solver's order."""
    t = np.linspace(t_start, t_end, n + 1)
    log_ac = -(beta_start * t + (beta_end - beta_start) * t ** 2 / (2.0 * (train_steps - 1)))
    ac = np.exp(log_ac)
    return np.sqrt(ac), np.sqrt(1.0 - ac)
