"""torch.optim.Adam's update with its amsgrad, maximize and decoupled_weight_decay options, restated in float64 in the
order of torch's _single_tensor_adam, with the gradient scaled first (the fused step's grad_scale):

    g = grad * scale;                      MAXIMIZE: g = -g
    wd != 0:  DECOUPLED: p = p * (1 - lr wd)     otherwise: g = g + wd p
    m = lerp(m, g, 1 - b1);  v = b2 v + (1 - b2) g^2
    AMSGRAD:  vmax = maximum(vmax, v)      (NaN where either is NaN, as torch.maximum)
    denom = sqrt(AMSGRAD ? vmax : v) / sqrt(1 - b2^t) + eps;  p = p - lr / (1 - b1^t) * m / denom

Flags are the C ABI's ELD_ADAM_* bits.  With none set this is tests/elementwise_ref.adam."""
import numpy as np

AMSGRAD, MAXIMIZE, DECOUPLED = 1, 2, 4
FLAG_SETS = tuple(range(8))


def maximum(a, b):
    """torch.maximum: NaN where either operand is NaN (numpy's np.maximum does the same)"""
    return np.maximum(a, b)


def adam(p, g, m, v, vmax, step, lr, beta1, beta2, eps, wd, scale, flags):
    """-> dict(p, m, v, vmax, Sp, Sm, Sv, Dp): the updated values in float64 (vmax as given where AMSGRAD is off) and
    the error rule's magnitudes: Sp = lr / bc1 |m'| / denom the size of the Adam update, Sm and Sv the magnitudes of the
    moment updates' terms, and Dp the absolute error that DECOUPLED's fp32 factor 1 - lr wd (rounded once: at most
    2^-24 off) and the product p (1 - lr wd) (rounded once more) can add, 2^-23 |p|."""
    with np.errstate(invalid='ignore'):                  # NaN and Inf gradients give NaN where torch gives NaN
        return _adam(p, g, m, v, vmax, step, lr, beta1, beta2, eps, wd, scale, flags)


def _adam(p, g, m, v, vmax, step, lr, beta1, beta2, eps, wd, scale, flags):
    p, g, m, v = (np.asarray(a, np.float64) for a in (p, g, m, v))
    vmax = None if vmax is None else np.asarray(vmax, np.float64)
    g = g * scale
    if flags & MAXIMIZE:
        g = -g
    dp = np.zeros_like(p)
    if wd != 0:
        if flags & DECOUPLED:
            dp = 2.0 ** -23 * np.abs(p)
            p = p * (1.0 - lr * wd)
        else:
            g = g + wd * p
    m1 = m + (1.0 - beta1) * (g - m)                     # exp_avg.lerp_(grad, 1 - beta1)
    v1 = v * beta2 + (1.0 - beta2) * (g * g)             # exp_avg_sq.mul_(beta2).addcmul_(grad, grad, value=1 - beta2)
    bc1 = 1.0 - beta1 ** step
    bc2 = 1.0 - beta2 ** step
    if flags & AMSGRAD:
        vmax = maximum(vmax, v1)
        denom = np.sqrt(vmax) / np.sqrt(bc2) + eps
    else:
        denom = np.sqrt(v1) / np.sqrt(bc2) + eps
    step_size = lr / bc1
    p1 = p - step_size * (m1 / denom)                    # param.addcdiv_(exp_avg, denom, value=-step_size)
    return dict(p=p1, m=m1, v=v1, vmax=vmax, Sp=step_size * np.abs(m1) / denom,
                Sm=np.abs(beta1 * m) + np.abs((1.0 - beta1) * g), Sv=np.abs(beta2 * v) + np.abs((1.0 - beta2) * g * g),
                Dp=dp)
