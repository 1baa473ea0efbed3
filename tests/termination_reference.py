"""numpy restatement of the early-termination decision of render(..., early_termination=t) (nrn_field_forward_terminate).

A pass's samples 0..S-1 are split into segments of K.  After segment r every ray still alive updates
T <- T * (1 - alpha_i + 1e-10) over the segment's samples, in order, in fp32 with one rounded operation per step, from
T = 1; the ray dies when T < t, and its termination_index is the end of that segment (S if it never dies).  alpha is the
pass's composite alpha output: compositing's own alphas, so the restatement reproduces the kernel bit for bit.  A dead
ray's later alphas are 0 (raw 0) and are never read."""
import numpy as np


def termination_index(alpha, K: int, t: float) -> np.ndarray:
    """alpha [N, S] (the composite alpha of the pass), K samples per segment, threshold t -> termination_index [N] int32."""
    alpha = np.ascontiguousarray(alpha, np.float32)
    n, S = alpha.shape
    one, eps, thr = np.float32(1.0), np.float32(1e-10), np.float32(t)
    T = np.ones(n, np.float32)
    out = np.full(n, S, np.int32)
    alive = np.ones(n, bool)
    for s0 in range(0, S, K):
        s1 = min(s0 + K, S)
        for i in range(s0, s1):
            om = (one - alpha[:, i]) + eps                     # two fp32 roundings, as (1 - alpha) + 1e-10 in the kernel
            T = np.where(alive, T * om, T).astype(np.float32)  # one rounded multiply
        with np.errstate(invalid="ignore"):
            die = alive & (T < thr)                            # NaN < t is false: a NaN T never dies
        out[die] = s1
        alive &= ~die
    return out


def transmittance_at_death(alpha, K: int, t: float) -> np.ndarray:
    """The fp32 T of each ray at the end of the segment in which it died (its running T after the last segment if it never
    died): the bound on how far rgb and acc can move."""
    alpha = np.ascontiguousarray(alpha, np.float32)
    n, S = alpha.shape
    idx = termination_index(alpha, K, t)
    one, eps = np.float32(1.0), np.float32(1e-10)
    T = np.ones(n, np.float32)
    for i in range(S):
        om = (one - alpha[:, i]) + eps
        T = np.where(i < idx, T * om, T).astype(np.float32)
    return T
