"""float32 restatement of the tf.train optimizer updates the fused training step runs (csrc/misc_kernels.cu opt_update), in the
kernel's operation order: every intermediate is np.float32 and rounded once per operation, so a replay over the trainer's own
gradients is bit-exact.  rsqrt(x) is 1 / sqrt(x), both correctly rounded.  The rules follow TF's training_ops functors as
remembered (DESIGN.md section 3): they are not verified against TensorFlow.

Each rule is ``step(p, g, slots, lr, hp) -> (p, slots)`` with ``slots`` a tuple in TF's creation order and ``hp`` the
aae_optimizer.hp entries of the rule.  ``adam`` restates the kernel's Adam (two fused multiply-adds, emulated by ``fma32``) for a
bit-exact replay; oracle.aae_oracle.tf_adam_step is TF's formula in float64 intermediates."""
import numpy as np

f32 = np.float32
ONE = f32(1)


def _rsqrt(x):
    return ONE / np.sqrt(x)


def fma32(a, b, c):
    """float32 fused multiply-add a * b + c with ONE rounding, elementwise.  The float64 product of two float32 values is exact;
    the float64 sum s of it and c is rounded, and its error e is recovered exactly (TwoSum).  Rounding s to float32 is then right
    except where s sits exactly on a float32 midpoint with e != 0: there the exact sum lies on e's side of the midpoint."""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    p = a.astype(np.float64) * b.astype(np.float64)
    c64 = c.astype(np.float64)
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    r = s.astype(np.float32)
    r64 = r.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        # the float32 neighbour of r on s's side; s is the midpoint of the two when it is halfway
        other = np.nextafter(r, np.where(s > r64, np.float32(np.inf), np.float32(-np.inf)).astype(np.float32))
        tie = (s != r64) & (s == (r64 + other.astype(np.float64)) * 0.5) & (e != 0)
        # ties-to-even picked r; the exact sum lies past the midpoint, at `other`'s side, when e points from r towards s
        r = np.where(tie & (np.sign(e) == np.sign(s - r64)), other, r)
    return r.astype(np.float32)


def adam(p, g, slots, lr_t, hp=(0.9, 0.999, 1e-8)):
    """The kernel's Adam, lr_t = lr sqrt(1 - b2^t) / (1 - b1^t) rounded once to float32 (as aae_train_step forms it on the host):
    m = fma(g, 1 - b1, b1 m); v = fma(g, (1 - b2) g, b2 v); var -= (lr_t m) / (sqrt(v) + eps).  TF's ApplyAdam in Eigen is the same
    formula; oracle.aae_oracle.tf_adam_step restates it in float64 intermediates, this one rounds where the kernel does."""
    m, v = slots
    b1, b2, eps = f32(hp[0]), f32(hp[1]), f32(hp[2])
    m = fma32(g, ONE - b1, b1 * m)
    v = fma32(g, (ONE - b2) * g, b2 * v)
    return p - (f32(lr_t) * m) / (np.sqrt(v) + eps), (m, v)


def adam_lr_t(lr, t, b1=0.9, b2=0.999):
    """Adam's bias-corrected step size after t updates, as aae_train_step computes it: double arithmetic on the float32 hp, one
    rounding to float32"""
    b1, b2 = float(f32(b1)), float(f32(b2))
    return f32(float(f32(lr)) * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t))


def gradient_descent(p, g, slots, lr, hp=()):
    """var -= grad * lr  (also ProximalGradientDescent with l1 = l2 = 0: the divisor 1 + l2 lr is exactly 1)"""
    return p - g * f32(lr), ()


def proximal_gradient_descent(p, g, slots, lr, hp=()):
    """TF's ApplyProximalGradientDescent at l1 = l2 = 0, written out: (var - grad lr) / (1 + l2 lr)"""
    lr, l2 = f32(lr), f32(0)
    return (p - g * lr) / (ONE + l2 * lr), ()


def adagrad(p, g, slots, lr, hp=(0.1,)):
    """accum += grad^2; var -= (grad * lr) * rsqrt(accum)"""
    (accum,) = slots
    accum = accum + g * g
    return p - (g * f32(lr)) * _rsqrt(accum), (accum,)


def proximal_adagrad(p, g, slots, lr, hp=(0.1,)):
    """accum += grad^2; lr_t = lr * rsqrt(accum); var = (var - grad * lr_t) / (1 + l2 lr_t) with l2 = 0, so / 1"""
    (accum,) = slots
    accum = accum + g * g
    lr_t = f32(lr) * _rsqrt(accum)
    return p - g * lr_t, (accum,)


def adadelta(p, g, slots, lr, hp=(0.95, 1e-8)):
    """accum = accum rho + grad^2 (1 - rho); upd = (sqrt(accum_update + eps) * rsqrt(accum + eps)) * grad; var -= upd * lr;
    accum_update = accum_update rho + upd^2 (1 - rho)"""
    accum, accum_update = slots
    rho, eps = f32(hp[0]), f32(hp[1])
    c = ONE - rho
    accum = accum * rho + (g * g) * c
    upd = (np.sqrt(accum_update + eps) * _rsqrt(accum + eps)) * g
    p = p - upd * f32(lr)
    accum_update = accum_update * rho + (upd * upd) * c
    return p, (accum, accum_update)


def rmsprop(p, g, slots, lr, hp=(0.9, 0.0, 1e-10)):
    """ms += (grad^2 - ms) (1 - decay); mom = mom momentum + (grad lr) / sqrt(ms + eps); var -= mom"""
    ms, mom = slots
    decay, momentum, eps = f32(hp[0]), f32(hp[1]), f32(hp[2])
    ms = ms + (g * g - ms) * (ONE - decay)
    mom = mom * momentum + (g * f32(lr)) / np.sqrt(ms + eps)
    return p - mom, (ms, mom)


def ftrl(p, g, slots, lr, hp=(0.1,)):
    """learning_rate_power -0.5, l1 = l2 = 0:  new = accum + grad^2; linear += grad - ((sqrt(new) - sqrt(accum)) / lr) var;
    var = |linear| > l1 ? (l1 sign(linear) - linear) / (sqrt(new) / lr + 2 l2) : 0; accum = new"""
    accum, linear = slots
    lr = f32(lr)
    new = accum + g * g
    sq = np.sqrt(new)
    linear = linear + (g - ((sq - np.sqrt(accum)) / lr) * p)
    with np.errstate(divide="ignore", invalid="ignore"):
        p = np.where(np.abs(linear) > f32(0), (-linear) / (sq / lr), f32(0)).astype(f32)
    return p, (new, linear)


RULES = {1: gradient_descent, 2: adagrad, 3: proximal_adagrad, 4: adadelta, 5: rmsprop, 6: ftrl}   # aae_optimizer_kind -> step
