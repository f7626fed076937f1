"""Float64 restatement of UniPC (Zhao et al. 2023, "UniPC: A Unified Predictor-Corrector Framework for Fast Sampling of
Diffusion Models", Algorithms 1-2) with data prediction and B(h) = bh2, in the step order of diffusers'
UniPCMultistepScheduler.step (diffusers is not a dependency: that order is restated here, not pinned against it).

Test infrastructure, like tests/dpm_oracle.py: it restates the paper, not the reference (which has no UniPC).  The product's
path is kandinsky2/model/gaussian_diffusion.py: UniPCSchedule / unipc_rows (one linear row per step) + k2_unipc_step; here each
step is written in the paper's form instead, with the R rho = b system solved by numpy at every step.

One step k of an N-step run from grid point `first`, with D_k = (x_k - sigma_k eps(x_k, k)) / alpha_k:
  UniC (k > first): re-solve the interval [k-1, k] from the previous CORRECTED sample `last` with the order p of the
      predictor that produced x_k, now that D_k is known:  x_k^c = sigma_k / sigma_{k-1} last - alpha_k phi D_{k-1}
      - alpha_k B(h) (sum_i rho_i D1_i + rho_p (D_k - D_{k-1})),  phi = B(h) = e^{-h} - 1 (bh2),  rho_p = 1/2 when p = 1.
      The current latent x_k only feeds the model.
  UniP: x_{k+1} = sigma_{k+1} / sigma_k x_k^c - alpha_{k+1} phi D_k - alpha_{k+1} B(h) sum_i rho_i D1_i  (rho = 1/2 at p = 2),
      order p = min(order, steps run so far + 1, N - k when lower_order_final).
  The history keeps D_k of the uncorrected x_k; `last` becomes x_k^c.
"""
import numpy as np


def _lam(alpha, sigma):
    with np.errstate(divide="ignore"):
        return np.log(np.asarray(alpha, dtype=np.float64)) - np.log(np.asarray(sigma, dtype=np.float64))


def _system(h, rks):
    """The paper's R rho = b system for B(h) = bh2 (data prediction, hh = -h): -> (R [p, p], b [p], phi_1 = e^{-h} - 1, B(h))."""
    hh = -h
    h_phi_1 = np.expm1(hh)
    h_phi_k = h_phi_1 / hh - 1.0
    b_h = np.expm1(hh)
    R, b, fac = [], [], 1.0
    for i in range(1, len(rks) + 1):
        R.append(rks ** (i - 1))
        b.append(h_phi_k * fac / b_h)
        fac *= i + 1
        h_phi_k = h_phi_k / hh - 1.0 / fac
    return np.array(R), np.array(b), h_phi_1, b_h


def solve(eps_fn, x, alpha, sigma, first=0, order=2, corrector=True, lower_order_final=True, inpaint=None,
          inpaint_renoise=True):
    """UniPC from x at grid point `first` to grid point n = len(alpha) - 1.  eps_fn(x, k) -> the (guided) epsilon at grid point
    k.  corrector=False is UniP alone (order 2: DPM-Solver++(2M)).  inpaint = (init, mask, noise0): inpaint_renoise=True is
    Kandinsky 2.2's rule (after every step the known region of x is init noised to the next grid point with noise0; `last` is
    not blended), False is 2.1's (the known region replaces D).  Works on numpy arrays and torch tensors alike."""
    n = len(alpha) - 1
    lam = [float(v) for v in _lam(alpha, sigma)]
    alpha, sigma = [float(v) for v in alpha], [float(v) for v in sigma]
    D, last, last_order = {}, None, None
    for k in range(first, n):
        d = (x - sigma[k] * eps_fn(x, k)) / alpha[k]
        if inpaint is not None and not inpaint_renoise:
            init, mask, _ = inpaint
            d = mask * init + (1 - mask) * d
        xc = x
        if corrector and last is not None:
            p, h = last_order, lam[k] - lam[k - 1]
            rks = np.array([(lam[k - 1 - i] - lam[k - 1]) / h for i in range(1, p)] + [1.0])
            R, b, h_phi_1, b_h = _system(h, rks)
            rhos = np.array([0.5]) if p == 1 else np.linalg.solve(R, b)
            corr = 0.0
            for i in range(1, p):
                corr = corr + float(rhos[i - 1]) * (D[k - 1 - i] - D[k - 1]) / float(rks[i - 1])
            xc = (sigma[k] / sigma[k - 1] * last - alpha[k] * float(h_phi_1) * D[k - 1]
                  - alpha[k] * float(b_h) * (corr + float(rhos[-1]) * (d - D[k - 1])))
        D[k] = d
        p = min(order, k - first + 1)
        if lower_order_final:
            p = min(p, n - k)
        h = lam[k + 1] - lam[k]
        rks = np.array([(lam[k - i] - lam[k]) / h for i in range(1, p)] + [1.0])
        with np.errstate(invalid="ignore"):
            R, b, h_phi_1, b_h = _system(h, rks)
        xn = sigma[k + 1] / sigma[k] * xc - alpha[k + 1] * float(h_phi_1) * d
        if p >= 2:
            rhos = np.array([0.5]) if p == 2 else np.linalg.solve(R[:-1, :-1], b[:-1])
            pred = 0.0
            for i in range(1, p):
                pred = pred + float(rhos[i - 1]) * (D[k - i] - d) / float(rks[i - 1])
            xn = xn - alpha[k + 1] * float(b_h) * pred
        if inpaint is not None and inpaint_renoise:
            init, mask, noise0 = inpaint
            xn = mask * (alpha[k + 1] * init + sigma[k + 1] * noise0) + (1 - mask) * xn
        last, last_order, x = xc, p, xn
    return x


def apply_rows(table, eps_fn, x, step_index=None, inpaint=None, inpaint_renoise=True):
    """k2_unipc_step's formula evaluated row by row in float64 (table: step-order rows of 16), each operand read only when its
    coefficient is non-zero:
        D = c0 x - c1 eps;  xc = a_x x + a_L last + a_0 D + a_1 D_{k-1} + a_2 D_{k-2};  x' = b_c xc + b_0 D + b_1 D_{k-1};
        last = xc;  (D_{k-2}, D_{k-1}) = (D_{k-1}, D)."""
    last = h1 = h2 = None
    for j, row in enumerate(table):
        k = j if step_index is None else step_index[j]
        d = row[0] * x - row[1] * eps_fn(x, k)
        if inpaint is not None and not inpaint_renoise:
            init, mask, _ = inpaint
            d = mask * init + (1 - mask) * d
        xc = row[4] * d
        for c, v in ((row[2], x), (row[3], last), (row[5], h1), (row[6], h2)):
            if c != 0.0:
                xc = xc + c * v
        xn = row[7] * xc + row[8] * d
        if row[9] != 0.0:
            xn = xn + row[9] * h1
        if inpaint is not None and inpaint_renoise:
            init, mask, noise0 = inpaint
            xn = mask * (row[10] * init + row[11] * noise0) + (1 - mask) * xn
        last, h2, h1, x = xc, h1, d, xn
    return x
