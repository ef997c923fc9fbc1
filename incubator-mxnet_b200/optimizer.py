"""Optimizer descriptors mirroring python/mxnet/optimizer/{optimizer,sgd,nag,adam,adamW,adabelief,rmsprop,signum,
ftml,adamax,adadelta,nadam,updater}.py.

Two roles:
* describe the hyper-parameters of the optimizers that have a fused kernel in the native
  engine (SGD / SGD-momentum / multi-precision SGD, NAG, Adam, AdamW, AdaBelief, RMSProp, Signum, FTML, Adamax,
  AdaDelta, Nadam, Test, and the layer-wise adaptive LAMB / LANS / LARS) -- ``KVStore.set_optimizer``
  hands them to ``MXKVB200SetOptimizer`` and the update then runs inside the reduce kernel;
* provide the generic ``Updater`` callback (updater.py:39-93) for any other Optimizer object:
  the store reduces on the GPU and calls back into Python, exactly like the reference.  The
  non-fused ``step`` arithmetic below runs as torch ops on the caller's stream.
"""
import math
import pickle

import numpy as np

from .ndarray import NDArray


class Optimizer(object):
    """Base class (python/mxnet/optimizer/optimizer.py:37-352): rescale_grad, clip_gradient,
    learning rate (+ scheduler), wd, per-index lr/wd multipliers and update counts."""
    opt_registry = {}
    fused_name = None

    def __init__(self, rescale_grad=1., param_idx2name=None, wd=0., clip_gradient=None, learning_rate=None,
                 lr_scheduler=None, begin_num_update=0, multi_precision=False, param_dict=None,
                 aggregate_num=None, use_fused_step=None, **kwargs):
        self.rescale_grad = rescale_grad
        self.lr_scheduler = lr_scheduler
        if self.lr_scheduler is None and learning_rate is None:
            learning_rate = 0.01
        self.lr = learning_rate
        # an explicit learning rate overrides the scheduler's base (optimizer.py:96-105); none leaves it alone
        if self.lr_scheduler is not None and learning_rate is not None:
            self.lr_scheduler.base_lr = learning_rate
        self.wd = wd
        self.lr_mult = {}
        self.wd_mult = {}
        self.begin_num_update = begin_num_update
        self.num_update = begin_num_update
        self._all_index_update_counts = {0: {}}          # per device id (optimizer.py:113-114)
        self._index_update_count = self._all_index_update_counts[0]
        self.clip_gradient = clip_gradient
        self.multi_precision = multi_precision
        self.aggregate_num = 1 if aggregate_num is None else aggregate_num      # optimizer.py:118-121
        if use_fused_step is not None:
            self.use_fused_step = use_fused_step
        self.idx2name = dict(param_idx2name or {})
        self.param_dict = param_dict or {}

    def __getstate__(self):
        """optimizer.py:544-553: ``param_dict`` (the Parameter objects) is not part of a saved optimizer; the
        Trainer attaches its own parameters again after loading."""
        ret = self.__dict__.copy()
        ret.pop("param_dict", None)
        return ret

    def __setstate__(self, state):
        self.__dict__ = state
        self.param_dict = {}

    @staticmethod
    def register(klass):
        Optimizer.opt_registry[klass.__name__.lower()] = klass
        return klass

    @staticmethod
    def create_optimizer(name, **kwargs):
        if name.lower() in Optimizer.opt_registry:
            return Optimizer.opt_registry[name.lower()](**kwargs)
        raise ValueError("Cannot find optimizer %s" % name)

    @property
    def learning_rate(self):
        if self.lr_scheduler is not None:
            return self.lr_scheduler(self.num_update)
        return self.lr

    def set_learning_rate(self, lr):
        if self.lr_scheduler is not None:
            raise UserWarning("LRScheduler of the optimizer has already been defined.")
        self.lr = lr

    def set_lr_mult(self, args_lr_mult):
        self.lr_mult = dict(args_lr_mult)

    def set_wd_mult(self, args_wd_mult):
        self.wd_mult = dict(args_wd_mult)

    def _set_current_context(self, device_id):
        """optimizer.py:433-443: one table of update counts per device, so that the per-device updaters of a
        Trainer that share this optimizer count every step once, not once per device."""
        if device_id not in self._all_index_update_counts:
            self._all_index_update_counts[device_id] = {}
        self._index_update_count = self._all_index_update_counts[device_id]

    def _update_count(self, index):
        """optimizer.py:445-462; ``index`` may be a list"""
        for idx in (index if isinstance(index, (list, tuple)) else [index]):
            self._index_update_count[idx] = self._index_update_count.get(idx, self.begin_num_update) + 1
            self.num_update = max(self._index_update_count[idx], self.num_update)

    def _get_lrs(self, indices):
        return [self._get_lr(i) for i in indices]

    def _get_wds(self, indices):
        return [self._get_wd(i) for i in indices]

    def _mult(self, table, attr, index):
        """Per-parameter multiplier in the reference's order of precedence (optimizer.py:479-487,518-525):
        the Parameter object, then the table by index, then the table by name."""
        if index in self.param_dict:
            return getattr(self.param_dict[index], attr, 1.0)
        if index in table:
            return table[index]
        if index in self.idx2name:
            return table.get(self.idx2name[index], 1.0)
        return 1.0

    def _get_lr(self, index):
        return self.learning_rate * self._mult(self.lr_mult, "lr_mult", index)

    def _get_wd(self, index):
        return self.wd * self._mult(self.wd_mult, "wd_mult", index)

    def key_multipliers(self):
        """{index or name: (lr_mult, wd_mult)} for every parameter whose multipliers differ from 1 -- what
        ``KVStore.set_optimizer`` hands to the engine (MXKVB200SetOptimizerMult)."""
        names = set(self.idx2name.values())
        keys = set(self.idx2name) | set(self.param_dict)
        for table in (self.lr_mult, self.wd_mult):
            for k in table:
                if not (isinstance(k, str) and k in names):      # names are reached through their index
                    keys.add(k)
        out = {}
        for k in keys:
            lm, wm = self._mult(self.lr_mult, "lr_mult", k), self._mult(self.wd_mult, "wd_mult", k)
            if lm != 1.0 or wm != 1.0:
                out[k] = (lm, wm)
        return out

    # hyper-parameters handed to the native fused kernel
    def fused_kwargs(self):
        kw = {"learning_rate": self.learning_rate, "wd": self.wd, "rescale_grad": self.rescale_grad,
              "multi_precision": bool(self.multi_precision)}
        if self.clip_gradient is not None:
            kw["clip_gradient"] = self.clip_gradient
        return kw

    # ---- the non-fused path: the reference's protocol for optimizers written in Python (optimizer.py:214-352),
    # which is what a user-defined Optimizer subclass implements.  Everything takes LISTS; ``step`` counts the
    # update itself (``self._update_count(indices)``) before it reads learning rates.
    use_fused_step = False

    def create_state(self, index, weight):
        return None

    def create_state_multi_precision(self, index, weight):
        """optimizer.py:214-243: a float32 master copy in front of the state for float16 weights"""
        if self.multi_precision and weight.dtype == np.float16:
            master = weight.astype(np.float32)
            return (master, self.create_state(index, master))
        return self.create_state(index, weight)

    def step(self, indices, weights, grads, states):
        raise NotImplementedError()

    def fused_step(self, indices, weights, grads, states):
        # the operator-backed flavour of the reference; in this package the fused kernels live in the engine
        # (fused_name), so on the Python path it is the same as step
        self.step(indices, weights, grads, states)

    def update(self, indices, weights, grads, states):
        """optimizer.py:287-318"""
        if not self.use_fused_step:
            self.step(indices, weights, grads, states)
        else:
            self.fused_step(indices, weights, grads, states)

    def update_multi_precision(self, indices, weights, grads, states):
        """optimizer.py:320-352"""
        masters, inner, grads32 = [], [], []
        for weight, grad, state in zip(weights, grads, states):
            if self.multi_precision and weight.dtype == np.float16:
                masters.append(state[0])
                inner.append(state[1])
                grads32.append(grad.astype(np.float32))
            else:
                masters.append(weight)
                inner.append(state)
                grads32.append(grad)
        self.update(indices, masters, grads32, inner)
        for master, weight in zip(masters, weights):
            if self.multi_precision and weight.dtype == np.float16:
                weight[:] = master.asnumpy().astype(np.float16)


register = Optimizer.register
create = Optimizer.create_optimizer


def _prep_grad(opt, index, w, g):
    import torch
    g = g.to(torch.float32) * opt.rescale_grad
    if opt.clip_gradient is not None:
        g = torch.clamp(g, -opt.clip_gradient, opt.clip_gradient)
    return g + opt._get_wd(index) * w


@register
class SGD(Optimizer):
    """python/mxnet/optimizer/sgd.py; fused kernels sgd_update / sgd_mom_update / mp_sgd_*."""
    fused_name = "sgd"

    def __init__(self, learning_rate=0.1, momentum=0.0, lazy_update=False, multi_precision=False, **kwargs):
        super(SGD, self).__init__(learning_rate=learning_rate, multi_precision=multi_precision, **kwargs)
        self.momentum = momentum
        self.lazy_update = lazy_update

    def fused_kwargs(self):
        kw = super(SGD, self).fused_kwargs()
        kw["momentum"] = self.momentum
        kw["lazy_update"] = bool(self.lazy_update)
        return kw

    def create_state(self, index, weight):
        import torch
        return torch.zeros_like(weight.as_torch(), dtype=torch.float32) if self.momentum != 0.0 else None

    def step(self, indices, weights, grads, states):     # sgd.py:118-154
        self._update_count(indices)
        lrs = self._get_lrs(indices)
        for index, weight, grad, state, lr in zip(indices, weights, grads, states, lrs):
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            if state is not None:
                state.mul_(self.momentum).sub_(lr * g)
                w.add_(state)
            else:
                w.sub_(lr * g)


@register
class NAG(Optimizer):
    """python/mxnet/optimizer/nag.py: Nesterov accelerated gradient; fused kernels nag_mom_update /
    mp_nag_mom_update (src/operator/optimizer_op-inl.h:1029-1092), sgd_update / mp_sgd_update at momentum 0::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        mom = momentum * mom - lr * grad
        weight = weight + momentum * mom - lr * grad
    """
    fused_name = "nag"

    def __init__(self, learning_rate=0.1, momentum=0.9, multi_precision=False, **kwargs):
        super(NAG, self).__init__(learning_rate=learning_rate, multi_precision=multi_precision, **kwargs)
        self.momentum = momentum

    def fused_kwargs(self):
        kw = super(NAG, self).fused_kwargs()
        kw["momentum"] = self.momentum
        return kw

    def create_state(self, index, weight):
        import torch
        return torch.zeros_like(weight.as_torch(), dtype=torch.float32) if self.momentum != 0.0 else None

    def step(self, indices, weights, grads, states):     # nag.py:72-109
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            if state is not None:
                state.mul_(self.momentum).sub_(lr * g)
                d = self.momentum * state - lr * g
            else:
                d = -lr * g
            w.add_(d)


@register
class Adam(Optimizer):
    """python/mxnet/optimizer/adam.py; fused kernel adam_update."""
    fused_name = "adam"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, lazy_update=False, **kwargs):
        super(Adam, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon, self.lazy_update = beta1, beta2, epsilon, lazy_update

    def fused_kwargs(self):
        kw = super(Adam, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon, lazy_update=bool(self.lazy_update))
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return (torch.zeros_like(w, dtype=torch.float32), torch.zeros_like(w, dtype=torch.float32))

    def step(self, indices, weights, grads, states):     # adam.py:107-147
        import torch
        self._update_count(indices)
        lrs = self._get_lrs(indices)
        for index, weight, grad, state, lr in zip(indices, weights, grads, states, lrs):
            w, g = weight.as_torch(), grad.as_torch()
            t = self._index_update_count[index]
            lr = lr * math.sqrt(1. - self.beta2 ** t) / (1. - self.beta1 ** t)
            g = _prep_grad(self, index, w, g)
            mean, var = state
            mean.mul_(self.beta1).add_((1. - self.beta1) * g)
            var.mul_(self.beta2).add_((1. - self.beta2) * g * g)
            w.sub_(lr * mean / (torch.sqrt(var) + self.epsilon))


@register
class AdamW(Optimizer):
    """python/mxnet/optimizer/adamW.py: ``w -= lr_t * (m / (sqrt(v) + eps) + wd * w)`` with
    ``lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t)`` (``correct_bias``).  The fused kernel is
    _adamw_update / _mp_adamw_update (src/operator/contrib/adamw-inl.h:101-124), driven the way the
    reference class drives it: operator ``lr = 1``, operator ``eta = lr_t`` (adamW.py:176-200).  ``eta`` here
    is an extra schedule multiplier of this engine (default 1); a ``rescale_grad`` of 0 / inf / nan skips the
    update like the operator does (adamw-inl.h:455)."""
    fused_name = "adamw"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6, correct_bias=True,
                 eta=1.0, **kwargs):
        super(AdamW, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon, self.eta = beta1, beta2, epsilon, eta
        self.correct_bias = correct_bias

    def fused_kwargs(self):
        kw = super(AdamW, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon, eta=self.eta,
                  correct_bias=bool(self.correct_bias))
        return kw


@register
class AdaBelief(Optimizer):
    """python/mxnet/optimizer/adabelief.py; fused kernels multi_adabelief_update / multi_mp_adabelief_update
    (src/operator/contrib/adabelief-inl.h:354-384), driven like AdamW: operator ``lr = 1``, operator
    ``eta = lr_t`` (adabelief.py:171-220), and a ``rescale_grad`` of 0 / inf / nan skips the update::

        grad = clip(grad * rescale_grad + wd * weight, clip_gradient)
        mean = beta1 * mean + (1 - beta1) * grad
        var = beta2 * var + (1 - beta2) * (grad - mean)**2 + epsilon
        lr_t = learning_rate * sqrt(1 - beta2**t) / (1 - beta1**t)      (correct_bias; else learning_rate)
        weight = weight - lr_t * mean / (sqrt(var) + epsilon)
    """
    fused_name = "adabelief"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6, correct_bias=True, **kwargs):
        super(AdaBelief, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.correct_bias = correct_bias

    def fused_kwargs(self):
        kw = super(AdaBelief, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon, correct_bias=bool(self.correct_bias))
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return (torch.zeros_like(w, dtype=torch.float32), torch.zeros_like(w, dtype=torch.float32))   # mean, var

    def step(self, indices, weights, grads, states):     # adabelief.py:112-139
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            t = self._index_update_count[index]
            w, g = weight.as_torch(), grad.as_torch()
            # weight decay BEFORE the clip (unlike _prep_grad's order)
            g = g.to(torch.float32) * self.rescale_grad + self._get_wd(index) * w
            if self.clip_gradient is not None:
                g = torch.clamp(g, -self.clip_gradient, self.clip_gradient)
            if self.correct_bias:
                lr *= math.sqrt(1. - self.beta2 ** t) / (1. - self.beta1 ** t)
            mean, var = state
            mean.mul_(self.beta1).add_((1. - self.beta1) * g)
            var.mul_(self.beta2).add_((1. - self.beta2) * torch.square(g - mean)).add_(self.epsilon)
            w.sub_(lr * (mean / (torch.sqrt(var) + self.epsilon)))


@register
class RMSProp(Optimizer):
    """python/mxnet/optimizer/rmsprop.py; fused kernels rmsprop_update (Tieleman & Hinton) and, with
    ``centered=True``, rmspropalex_update (Graves) (src/operator/optimizer_op-inl.h:1905-2031)::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        centered=False:  var = rho * var + (1 - rho) * grad**2
                         weight = weight - lr * grad / (sqrt(var) + epsilon)
        centered=True:   mean = rho * mean + (1 - rho) * grad;  var = rho * var + (1 - rho) * grad**2
                         mom = momentum * mom - lr * grad / sqrt(var - mean**2 + epsilon)
                         weight = weight + mom
        weight = clip(weight, clip_weights)

    As in ``RMSProp.fused_step`` (rmsprop.py:169-172), the fused update clips only where ``clip_gradient`` /
    ``clip_weights`` is truthy: 0, a negative value or None turns that clip off."""
    fused_name = "rmsprop"

    def __init__(self, learning_rate=0.001, rho=0.9, momentum=0.9, epsilon=1e-8, centered=False, clip_weights=None,
                 **kwargs):
        super(RMSProp, self).__init__(learning_rate=learning_rate, **kwargs)
        self.rho, self.momentum, self.epsilon = rho, momentum, epsilon
        self.centered, self.clip_weights = centered, clip_weights

    def fused_kwargs(self):
        kw = super(RMSProp, self).fused_kwargs()
        kw.update(rho=self.rho, momentum=self.momentum, epsilon=self.epsilon, centered=bool(self.centered),
                  clip_weights=self.clip_weights)
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        if self.centered:        # mean, var, mom
            return tuple(torch.zeros_like(w, dtype=torch.float32) for _ in range(3))
        return torch.zeros_like(w, dtype=torch.float32)      # var

    def step(self, indices, weights, grads, states):     # rmsprop.py:90-141
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            if not self.centered:
                var = state
                var.mul_(self.rho).add_((1 - self.rho) * torch.square(g))
                w.sub_(lr * (g / (torch.sqrt(var) + self.epsilon)))
            else:
                mean, var, mom = state
                mean.mul_(self.rho).add_((1 - self.rho) * g)
                var.mul_(self.rho).add_((1 - self.rho) * torch.square(g))
                mom.mul_(self.momentum).sub_(lr * g / torch.sqrt(var - torch.square(mean) + self.epsilon))
                w.add_(mom)
            if self.clip_weights:
                w.clamp_(-self.clip_weights, self.clip_weights)


def _sign(x):
    """(x > 0) - (x < 0), as signum.py writes it: NaN gives 0 (torch.sign gives NaN)"""
    return (x > 0).to(x.dtype) - (x < 0).to(x.dtype)


@register
class Signum(Optimizer):
    """python/mxnet/optimizer/signum.py: signSGD / Signum (Bernstein et al., 2018); fused kernels signsgd_update
    (no state, momentum 0) and signum_update (src/operator/optimizer_op-inl.h:2293-2379)::

        momentum == 0:  weight = (1 - lr * (wd + wd_lh)) * weight - lr * sign(grad)
        otherwise:      grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
                        mom = momentum * mom - (1 - momentum) * grad
                        weight = (1 - lr * wd_lh) * weight + lr * sign(mom)

    ``mom`` holds the negated average, as in the reference's state.  As in ``Signum.fused_step`` (signum.py:121-158),
    the fused signsgd_update takes the sign of the raw summed gradient (rescale_grad and clip_gradient do not enter),
    signum_update runs a negative momentum as 0, and a ``clip_gradient`` of 0, below 0 or None is off; ``wd_lh`` is
    not multiplied by ``wd_mult``."""
    fused_name = "signum"

    def __init__(self, learning_rate=0.01, momentum=0.9, wd_lh=0.0, **kwargs):
        super(Signum, self).__init__(learning_rate=learning_rate, **kwargs)
        self.momentum, self.wd_lh = momentum, wd_lh

    def fused_kwargs(self):
        kw = super(Signum, self).fused_kwargs()
        kw.update(momentum=self.momentum, wd_lh=self.wd_lh)
        return kw

    def create_state(self, index, weight):
        import torch
        return torch.zeros_like(weight.as_torch(), dtype=torch.float32) if self.momentum != 0.0 else None

    def step(self, indices, weights, grads, states):     # signum.py:80-119
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            wd = self._get_wd(index)
            w, g = weight.as_torch(), grad.as_torch().to(torch.float32)
            if state is not None:
                g = g * self.rescale_grad
                if self.clip_gradient is not None:
                    g = torch.clamp(g, -self.clip_gradient, self.clip_gradient)
                g = g + wd * w
                state.mul_(self.momentum).sub_((1 - self.momentum) * g)
                w.mul_(1 - lr * self.wd_lh).add_(lr * _sign(state))
            else:
                w.mul_(1 - lr * (wd + self.wd_lh)).sub_(lr * _sign(g))


@register
class FTML(Optimizer):
    """python/mxnet/optimizer/ftml.py: Follow the Moving Leader (Zheng & Kwok, 2017); fused kernel ftml_update
    (src/operator/optimizer_op-inl.h:1117-1206)::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        v = beta2 * v + (1 - beta2) * grad**2
        d_t = (1 - beta1**t) / lr * (sqrt(v / (1 - beta2**t)) + epsilon)
        z = beta1 * z + (1 - beta1) * grad - (d_t - beta1 * d) * weight
        d = d_t
        weight = -z / d_t

    As in ``FTML.fused_step`` (ftml.py:127-158), the fused update clips only where ``clip_gradient`` is truthy: 0, a
    negative value or None is off (the non-fused ``step`` clips at 0)."""
    fused_name = "ftml"

    def __init__(self, learning_rate=0.0025, beta1=0.6, beta2=0.999, epsilon=1e-8, **kwargs):
        super(FTML, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon

    def fused_kwargs(self):
        kw = super(FTML, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon)
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return tuple(torch.zeros_like(w, dtype=torch.float32) for _ in range(3))     # d, v, z

    def step(self, indices, weights, grads, states):     # ftml.py:80-125
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            t = self._index_update_count[index]
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            coef1 = 1. - self.beta1 ** t
            coef2 = 1. - self.beta2 ** t
            d, v, z = state
            v.mul_(self.beta2).add_((1. - self.beta2) * torch.square(g))
            sigma = -self.beta1 * d
            d.copy_(torch.sqrt(v / coef2) + self.epsilon).mul_(coef1 / lr)
            sigma = sigma + d
            z.mul_(self.beta1).add_((1. - self.beta1) * g).sub_(sigma * w)
            w.copy_(-z / d)


def _maximum(a, b):
    """mshadow_op::maximum (mshadow_op.h:1266-1275): NaN in either operand gives NaN, as torch.maximum does"""
    import torch
    return torch.maximum(a, b)


@register
class Adamax(Optimizer):
    """python/mxnet/optimizer/adamax.py: AdaMax, the infinity-norm variant of Adam (Kingma & Ba, 2014, section 7).
    The reference has no operator for it: the fused kernel restates ``Adamax.step`` (adamax.py:74-111) one float32
    operation per NDArray operation, every Python scalar rounded once from its double::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        mean = beta1 * mean + (1 - beta1) * grad
        var = maximum(beta2 * var, abs(grad))
        weight = weight - lr / (1 - beta1**t) * (mean / (var + epsilon))

    ``clip_gradient`` clips whenever it is not None, at 0 too; a negative one is off in the fused kernel."""
    fused_name = "adamax"

    def __init__(self, learning_rate=0.002, beta1=0.9, beta2=0.999, epsilon=1e-8, **kwargs):
        super(Adamax, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon

    def fused_kwargs(self):
        kw = super(Adamax, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon)
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return tuple(torch.zeros_like(w, dtype=torch.float32) for _ in range(2))     # mean, var

    def step(self, indices, weights, grads, states):     # adamax.py:74-111
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            t = self._index_update_count[index]
            lr /= (1. - self.beta1 ** t)
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            mean, var = state
            mean.mul_(self.beta1).add_((1. - self.beta1) * g)
            var.copy_(_maximum(self.beta2 * var, g.abs()))
            w.sub_(lr * (mean / (var + self.epsilon)))


@register
class AdaDelta(Optimizer):
    """python/mxnet/optimizer/adadelta.py: AdaDelta (Zeiler, 2012).  The reference has no operator for it: the fused
    kernel restates ``AdaDelta.step`` (adadelta.py:72-111) one float32 operation per NDArray operation, every Python
    scalar rounded once from its double::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        acc_g = rho * acc_g + (1 - rho) * grad**2
        delta = sqrt(acc_delta + epsilon) / sqrt(acc_g + epsilon) * grad
        acc_delta = rho * acc_delta + (1 - rho) * delta**2
        weight = weight - lr * delta

    ``clip_gradient`` clips whenever it is not None, at 0 too; a negative one is off in the fused kernel."""
    fused_name = "adadelta"

    def __init__(self, learning_rate=1.0, rho=0.9, epsilon=1e-6, **kwargs):
        super(AdaDelta, self).__init__(learning_rate=learning_rate, **kwargs)
        self.rho, self.epsilon = rho, epsilon

    def fused_kwargs(self):
        kw = super(AdaDelta, self).fused_kwargs()
        kw.update(rho=self.rho, epsilon=self.epsilon)
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return tuple(torch.zeros_like(w, dtype=torch.float32) for _ in range(2))     # acc_g, acc_delta

    def step(self, indices, weights, grads, states):     # adadelta.py:72-111
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            acc_g, acc_delta = state
            acc_g.mul_(self.rho).add_((1. - self.rho) * torch.square(g))
            delta = torch.sqrt(acc_delta + self.epsilon)
            delta = delta / torch.sqrt(acc_g + self.epsilon) * g
            acc_delta.mul_(self.rho).add_((1. - self.rho) * torch.square(delta))
            w.sub_(lr * delta)


@register
class Nadam(Optimizer):
    """python/mxnet/optimizer/nadam.py: Adam with Nesterov momentum (Dozat, 2016).  The reference has no operator for
    it: the fused kernel restates ``Nadam.step`` (nadam.py:74-124) one float32 operation per NDArray operation, every
    Python scalar rounded once from its double::

        grad = clip(grad * rescale_grad, clip_gradient) + wd * weight
        momentum_t   = beta1 * (1 - 0.5 * 0.96**(t * schedule_decay))
        momentum_t_1 = beta1 * (1 - 0.5 * 0.96**((t + 1) * schedule_decay))
        m_schedule   = m_schedule * momentum_t            (ONE product for the optimizer, advanced by every update)
        mean = beta1 * mean + (1 - beta1) * grad;  var = beta2 * var + (1 - beta2) * grad**2
        mean_bar = momentum_t_1 * mean / (1 - m_schedule * momentum_t_1) + (1 - momentum_t) * grad / (1 - m_schedule)
        weight = weight - lr * mean_bar / (sqrt(var / (1 - beta2**t)) + epsilon)

    ``m_schedule`` is handed to the store with the other hyper-parameters and read back after every fused update, so
    that it stands where the store's updates took it (a saved optimizer, a Python ``step`` taking over).
    ``clip_gradient`` clips whenever it is not None, at 0 too; a negative one is off in the fused kernel."""
    fused_name = "nadam"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, schedule_decay=0.004, **kwargs):
        super(Nadam, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.schedule_decay = schedule_decay
        self.m_schedule = 1.

    def fused_kwargs(self):
        kw = super(Nadam, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon, schedule_decay=self.schedule_decay,
                  m_schedule=self.m_schedule)
        return kw

    def create_state(self, index, weight):
        import torch
        w = weight.as_torch()
        return tuple(torch.zeros_like(w, dtype=torch.float32) for _ in range(2))     # mean, var

    def step(self, indices, weights, grads, states):     # nadam.py:74-124
        import torch
        for index, weight, grad, state in zip(indices, weights, grads, states):
            self._update_count(index)
            lr = self._get_lr(index)
            t = self._index_update_count[index]
            w, g = weight.as_torch(), grad.as_torch()
            g = _prep_grad(self, index, w, g)
            coef2 = 1. - self.beta2 ** t
            momentum_t = self.beta1 * (1. - 0.5 * (pow(0.96, t * self.schedule_decay)))
            momentum_t_1 = self.beta1 * (1. - 0.5 * (pow(0.96, (t + 1) * self.schedule_decay)))
            self.m_schedule = self.m_schedule * momentum_t
            m_schedule_next = self.m_schedule * momentum_t_1
            mean, var = state
            mean.mul_(self.beta1).add_((1. - self.beta1) * g)
            var.mul_(self.beta2).add_((1. - self.beta2) * torch.square(g))
            grad_prime = g / (1. - self.m_schedule)
            mean_prime = mean / (1. - m_schedule_next)
            var_prime = var / coef2
            mean_bar = momentum_t_1 * mean_prime + (1. - momentum_t) * grad_prime
            w.sub_(lr * (mean_bar / (torch.sqrt(var_prime) + self.epsilon)))


class _LayerwiseAdaptive(Optimizer):
    """Shared part of LAMB / LANS / LARS: ``skip_nonfinite=True`` asks the store to leave weights and
    state alone when a merged gradient holds inf/nan (the AMP overflow skip, gluon/trainer.py:445-448,
    decided on the device; query it with ``KVStore.overflow()``)."""

    def __init__(self, skip_nonfinite=False, **kwargs):
        super(_LayerwiseAdaptive, self).__init__(**kwargs)
        self.skip_nonfinite = skip_nonfinite

    def fused_kwargs(self):
        kw = super(_LayerwiseAdaptive, self).fused_kwargs()
        if self.skip_nonfinite:
            kw["skip_nonfinite"] = True
        return kw


@register
class LAMB(_LayerwiseAdaptive):
    """python/mxnet/optimizer/lamb.py; fused kernels multi_lamb_update / multi_mp_lamb_update
    (src/operator/contrib/multi_lamb.cc:36-120) with the two norms taken inside the gradient exchange."""
    fused_name = "lamb"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6, lower_bound=None,
                 upper_bound=None, bias_correction=True, aggregate_num=4, **kwargs):
        super(LAMB, self).__init__(learning_rate=learning_rate, aggregate_num=aggregate_num, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.lower_bound, self.upper_bound, self.bias_correction = lower_bound, upper_bound, bias_correction

    def fused_kwargs(self):
        kw = super(LAMB, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon,
                  bias_correction=bool(self.bias_correction))
        if self.lower_bound:            # lamb.py:182-185: falsy bounds are not passed
            kw["lower_bound"] = self.lower_bound
        if self.upper_bound:
            kw["upper_bound"] = self.upper_bound
        return kw


@register
class LANS(_LayerwiseAdaptive):
    """python/mxnet/optimizer/lans.py; fused kernels multi_lans_update / multi_mp_lans_update
    (src/operator/contrib/multi_lans.cc:36-130)."""
    fused_name = "lans"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-6, lower_bound=None,
                 upper_bound=None, **kwargs):
        kwargs.setdefault("aggregate_num", 4)                    # lans.py:63
        super(LANS, self).__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon
        self.lower_bound, self.upper_bound = lower_bound, upper_bound

    def fused_kwargs(self):
        kw = super(LANS, self).fused_kwargs()
        kw.update(beta1=self.beta1, beta2=self.beta2, epsilon=self.epsilon)
        if self.lower_bound:
            kw["lower_bound"] = self.lower_bound
        if self.upper_bound:
            kw["upper_bound"] = self.upper_bound
        return kw


@register
class LARS(_LayerwiseAdaptive):
    """python/mxnet/optimizer/lars.py: lr *= eta * ||w|| / (||g|| + wd * ||w|| + eps) per layer (not for
    names ending in gamma / beta / bias), then the sgd / sgd_mom update."""
    fused_name = "lars"

    def __init__(self, learning_rate=0.1, momentum=0.0, eta=0.001, epsilon=1e-8, **kwargs):
        super(LARS, self).__init__(learning_rate=learning_rate, **kwargs)
        self.momentum, self.eta, self.epsilon = momentum, eta, epsilon

    def fused_kwargs(self):
        kw = super(LARS, self).fused_kwargs()
        kw.update(momentum=self.momentum, eta=self.eta, epsilon=self.epsilon)
        return kw

    def no_trust_ratio_indices(self):
        """Indices whose name ends in gamma / beta / bias (lars.py:121-123)."""
        return [i for i, n in self.idx2name.items() if str(n).endswith(("gamma", "beta", "bias"))]


@register
class Test(Optimizer):
    """The Test optimizer (optimizer.py:561-577): w -= lr * (rescale_grad * g + wd * w)."""
    fused_name = "test"

    def create_state(self, index, weight):
        return None

    def step(self, indices, weights, grads, states):
        self._update_count(indices)
        for index, weight, grad in zip(indices, weights, grads):
            w, g = weight.as_torch(), grad.as_torch()
            w.sub_(self._get_lr(index) * (self.rescale_grad * g + self._get_wd(index) * w))


def _device_id(weight):
    ctx = getattr(weight, "context", None)
    return getattr(ctx, "device_id", 0) if ctx is not None else 0


class _SavedNDArray(object):
    """an engine array inside a pickled Updater state"""

    def __init__(self, value, dev_type, dev_id):
        self.value, self.dev_type, self.dev_id = value, dev_type, dev_id


class Updater(object):
    """The kvstore updater callback (python/mxnet/optimizer/updater.py:30-127)."""

    def __init__(self, optimizer):
        self.optimizer = optimizer
        self.states = {}
        self.states_synced = {}

    def __call__(self, index, grad, weight):
        """updater.py:39-93: single values or lists; states are created on first sight with
        ``create_state_multi_precision``; the optimizer's ``update_multi_precision`` does the rest (its
        ``step`` counts the update)."""
        if not isinstance(index, (list, tuple)):
            indices, grads, weights = [index], [grad], [weight]
        else:
            indices, grads, weights = list(index), list(grad), list(weight)
        if weights:
            self.optimizer._set_current_context(_device_id(weights[0]))  # updater.py:50-51
        for i, idx in enumerate(indices):
            if isinstance(idx, bytes):
                indices[i] = idx = idx.decode()
            if idx not in self.states:
                self.states[idx] = self.optimizer.create_state_multi_precision(idx, weights[i])
                self.states_synced[idx] = True
        self.optimizer.update_multi_precision(indices, weights, grads, [self.states[i] for i in indices])

    def get_states(self, dump_optimizer=False):
        def host(s):
            if s is None:
                return None
            if isinstance(s, (tuple, list)):
                return tuple(host(x) for x in s)
            if isinstance(s, NDArray):                       # e.g. a multi-precision master copy
                return _SavedNDArray(s.asnumpy(), s.context.device_typeid, s.context.device_id)
            if hasattr(s, "detach"):
                return s.detach().cpu().numpy()
            return s
        states = {k: host(v) for k, v in self.states.items()}
        return pickle.dumps((states, self.optimizer) if dump_optimizer else states)

    def set_states(self, states):
        import torch
        states = pickle.loads(states)
        if isinstance(states, tuple) and len(states) == 2 and isinstance(states[1], Optimizer):
            states, self.optimizer = states

        def dev(s):
            if s is None:
                return None
            if isinstance(s, tuple):
                return tuple(dev(x) for x in s)
            if isinstance(s, _SavedNDArray):
                from . import ndarray as _ndm
                from .context import Context
                return _ndm.array(s.value, Context(Context.devtype2str[s.dev_type], s.dev_id), dtype=s.value.dtype)
            if isinstance(s, np.ndarray):
                return torch.from_numpy(s)
            return s
        self.states = {k: dev(v) for k, v in states.items()}
        self.states_synced = dict.fromkeys(self.states, True)


_FUSED_METHODS = ("step", "fused_step", "update", "update_multi_precision", "create_state",
                  "create_state_multi_precision", "fused_kwargs")


def fused_name_of(optimizer):
    """Name of the engine's fused kernel for ``optimizer``, or None when the Python path must run:
    the class has no fused kernel, the caller asked for ``use_fused_step=False``
    (optimizer.py:287-318), or a user subclass overrides a method the fused kernel stands in for
    (its ``step`` would otherwise be silently ignored)."""
    name = getattr(optimizer, "fused_name", None)
    if not name:
        return None
    if optimizer.__dict__.get("use_fused_step", None) is False:
        return None
    cls = type(optimizer)
    owner = next((c for c in cls.__mro__ if c.__dict__.get("fused_name") == name), None)
    if owner is None:
        return None
    if cls is not owner:
        for m in _FUSED_METHODS:
            if getattr(cls, m, None) is not getattr(owner, m, None):
                return None
    return name


class NativeUpdater(object):
    """Same call contract as :class:`Updater` (updater.py:39-93; ``index`` / ``grad`` / ``weight`` may be
    lists), but the whole list is updated IN PLACE by one fused launch (sequence) of the native engine
    -- what the reference does with ``multi_sgd_mom_update`` / ``multi_mp_sgd_*`` / ``multi_adamw`` /
    ``multi_adabelief`` / ``rmsprop_update`` / ``signum_update`` / ``ftml_update`` / ``multi_lamb`` / ``multi_lans``, or
    ``Adamax.step`` / ``AdaDelta.step`` / ``Nadam.step`` (which have no operator), when parameters are not updated on the kvstore (sgd.py:170-213, lamb.py:170-215).  One instance serves one device, like
    ``Trainer._updaters[dev]``."""

    def __init__(self, optimizer):
        from . import kvstore as _kvs
        assert fused_name_of(optimizer), "no fused kernel for %s" % type(optimizer).__name__
        self.optimizer = optimizer
        self._kv = _kvs.KVStore("updater")
        self._kw = None
        self._pending = None          # states loaded before the indices are known to the engine
        self._sync()

    def _sync(self):
        kw = self.optimizer.fused_kwargs()
        kw.pop("learning_rate", None)
        kw.pop("m_schedule", None)    # (handed over around every call: __call__)
        if kw != self._kw:            # rescale_grad etc. changed (Trainer.step sets it per batch size)
            self._kv.set_optimizer(self.optimizer)
            self._kw = kw
        self._kv._sync_lr()

    def __call__(self, index, grad, weight):
        from .base import _LIB, check_call, c_str_array
        import ctypes
        if not isinstance(index, (list, tuple)):
            index, grad, weight = [index], [grad], [weight]
        self.optimizer._set_current_context(_device_id(weight[0]))       # updater.py:50-51
        for i in dict.fromkeys(index):   # count first, then read the learning rate (sgd.py:184-186)
            self.optimizer._update_count(i)
        self._sync()
        self._kv._sync_mults(index)
        before = {i: self.optimizer._index_update_count[i] - 1 for i in dict.fromkeys(index)
                  if i not in self._kv._synced}
        n = len(index)
        use_str = isinstance(index[0], str)
        wh = (ctypes.c_void_p * n)(*[w.handle.value for w in weight])
        gh = (ctypes.c_void_p * n)(*[g.handle.value for g in grad])
        keys = c_str_array(list(index)) if use_str else (ctypes.c_int * n)(*[int(i) for i in index])
        fn = _LIB.MXKVB200UpdaterStepEx if use_str else _LIB.MXKVB200UpdaterStep
        if self._pending is not None:
            have = [i for i in index if i in self._pending["states"]]
            if have:
                check_call(fn(self._kv.handle, n, keys, wh, None))          # register, then load
                self._kv._load_fused_states(self._pending, only=set(have))
                for i in have:
                    del self._pending["states"][i]
                    before[i] = self.optimizer._index_update_count[i] - 1
        if before:                       # the engine counts from where the optimizer stands (see KVStore._advance_counts)
            if not set(before) <= self._kv._keys:
                check_call(fn(self._kv.handle, n, keys, wh, None))          # make the indices known first
            for i, c in before.items():
                self._kv._set_count(i, c)
                self._kv._synced.add(i)
        # Nadam: the per-device updaters of a Trainer share one optimizer object and so one schedule product, which
        # each call advances once per pair in pair order; it travels through the object between the devices' stores
        nadam = self.optimizer.fused_name == "nadam"
        if nadam:
            if self.optimizer.aggregate_num > 1 and n > 1:
                # updater.py:65-80: an aggregating updater groups the pairs by dtype (first seen first) before it steps
                first = {}
                for w in weight:
                    first.setdefault(w.dtype, len(first))
                order = sorted(range(n), key=lambda i: first[weight[i].dtype])
                index, weight, grad = [index[i] for i in order], [weight[i] for i in order], [grad[i] for i in order]
                wh = (ctypes.c_void_p * n)(*[w.handle.value for w in weight])
                gh = (ctypes.c_void_p * n)(*[g.handle.value for g in grad])
                keys = c_str_array(list(index)) if use_str else (ctypes.c_int * n)(*[int(i) for i in index])
            self._kv._set_scalar("m_schedule", self.optimizer.m_schedule)
        check_call(fn(self._kv.handle, n, keys, wh, gh))
        self._kv._keys.update(index)
        if nadam:
            self.optimizer.m_schedule = self._kv._get_scalar("m_schedule")

    def get_states(self, dump_optimizer=False):
        return self._kv._dump_fused_states(dump_optimizer)

    def set_states(self, states):
        payload = pickle.loads(states)
        assert payload.get("format") == "mxkv_b200_fused_v1", "not a fused-optimizer state blob"
        if "optimizer" in payload:
            self.optimizer = payload["optimizer"]
            self._kw = None
        self._pending = {"format": payload["format"], "states": dict(payload["states"])}


def get_updater(optimizer, native=None):
    """updater.py:130-143.  ``native`` (default: whenever the optimizer has a fused kernel) selects the
    engine-side multi-tensor updater; otherwise the generic Python one."""
    if native is None:
        native = bool(fused_name_of(optimizer))
    return NativeUpdater(optimizer) if native else Updater(optimizer)
