"""Python KVStore front-end: same surface as python/mxnet/kvstore/{base,kvstore}.py.

* ``KVStoreBase`` + ``KVStoreBase.register`` + ``create(name)``: the plug-in registry
  (base.py:74-243, 406-461).  ``create`` looks the registry up first and falls back to the
  native store, like the reference.
* ``KVStore``: the native wrapper (kvstore.py:54-742): init / push / pull / pushpull /
  broadcast / row_sparse_pull / set_optimizer / _set_updater / save|load_optimizer_states /
  type / rank / num_workers / is_capable / set_gradient_compression / _barrier.

To let the reference's own ``mx.kv.create`` / ``gluon.Trainer`` pick this engine up, register
:class:`KVStore` subclasses with the reference's ``mx.kvstore.KVStoreBase.register`` (see
INTEGRATION.md); the method set below is exactly what that registry expects.
"""
import ctypes
import pickle

import numpy as np

from .base import _LIB, check_call, c_str, c_str_array, c_array, MXNetError, KVStoreHandle
from .ndarray import NDArray
from . import ndarray as _nd
from . import optimizer as opt
from operator import is_ as _is


def _ctype_key_value(keys, vals):
    """Flatten (keys, vals) key-major like base.py:32-65.  Returns (keys list, NDArray list,
    use_str_keys).  Written as a loop, not a recursion: a training step passes a few hundred keys and this
    sits on the host's critical path (the launch is asynchronous; the marshalling is not)."""
    if not isinstance(keys, (tuple, list)):
        assert isinstance(keys, (int, str)), "unexpected type for keys: " + str(type(keys))
        use_str = isinstance(keys, str)
        if isinstance(vals, NDArray):
            return [keys], [vals], use_str
        vals = list(vals)
        assert all(isinstance(v, NDArray) for v in vals)
        return [keys] * len(vals), vals, use_str
    assert len(keys) == len(vals)
    c_keys, c_vals = [], []
    n_str = 0
    for key, val in zip(keys, vals):
        if isinstance(key, (tuple, list)):                     # nested key lists: the general case
            k_i, v_i, s_i = _ctype_key_value(key, val)
            c_keys += k_i
            c_vals += v_i
            n_str += len(k_i) if s_i else 0
            continue
        if isinstance(key, str):
            n_str += 1 if isinstance(val, NDArray) else len(val)
        else:
            assert isinstance(key, int), "unexpected type for keys: " + str(type(key))
        if isinstance(val, NDArray):
            c_keys.append(key)
            c_vals.append(val)
        else:
            for v in val:
                assert isinstance(v, NDArray)
                c_keys.append(key)
                c_vals.append(v)
    assert n_str == 0 or n_str == len(c_keys), "inconsistent types of keys detected."
    return c_keys, c_vals, (n_str > 0 if c_keys else None)


def _c_keys(keys, use_str):
    return c_str_array(keys) if use_str else c_array(ctypes.c_int, keys)


def _c_vals(vals):
    arr = (ctypes.c_void_p * len(vals))()
    arr[:] = [v._h for v in vals]
    return arr


class KVStoreBase(object):
    """An abstract key-value store interface for data parallel training (base.py:74-243)."""
    OPTIMIZER = "optimizer"
    kv_registry = {}

    def broadcast(self, key, value, out, priority=0):
        raise NotImplementedError()

    def pushpull(self, key, value, out=None, priority=0):
        raise NotImplementedError()

    def set_optimizer(self, optimizer):
        raise NotImplementedError()

    def is_capable(self, capability):
        raise NotImplementedError()

    def save_optimizer_states(self, fname, dump_optimizer=False):
        raise NotImplementedError()

    def load_optimizer_states(self, fname):
        raise NotImplementedError()

    @property
    def type(self):
        raise NotImplementedError()

    @property
    def rank(self):
        raise NotImplementedError()

    @property
    def num_workers(self):
        raise NotImplementedError()

    @staticmethod
    def register(klass):
        assert isinstance(klass, type)
        KVStoreBase.kv_registry[klass.__name__.lower()] = klass
        return klass


class KVStore(KVStoreBase):
    """Native key-value store (kvstore.py:54-742) backed by libmxkv_b200.so."""

    def __init__(self, handle_or_name="device"):
        if isinstance(handle_or_name, str):
            handle = KVStoreHandle()
            check_call(_LIB.MXKVStoreCreate(c_str(handle_or_name), ctypes.byref(handle)))
            self.handle = handle
        else:
            self.handle = handle_or_name
        self._updater = None
        self._updater_func = None
        self._str_updater_func = None
        self._optimizer = None
        self._fused = False
        self._last_lr = None
        self._keys = set()
        self._mults = {}
        self._synced = set()

    def __del__(self):
        try:
            check_call(_LIB.MXKVStoreFree(self.handle))
        except Exception:
            pass

    # -- data path -------------------------------------------------------------
    def init(self, key, value):
        keys, vals, use_str = _ctype_key_value(key, value)
        fn = _LIB.MXKVStoreInitEx if use_str else _LIB.MXKVStoreInit
        check_call(fn(self.handle, len(keys), _c_keys(keys, use_str), _c_vals(vals)))
        self._keys.update(keys)

    def _advance_counts(self, keys):
        """Optimizer._update_count for every distinct pushed key, THEN the learning rate: the reference's
        fused_step counts first and asks the scheduler afterwards (sgd.py:184-186), so the first update
        already runs at ``lr_scheduler(1)``.  The engine keeps the same per-key counts (bias correction)."""
        if self._fused and self._optimizer is not None:
            opt_ = self._optimizer
            uniq = list(dict.fromkeys(keys))
            cnt, begin, top = opt_._index_update_count, opt_.begin_num_update, opt_.num_update
            synced = self._synced
            for k in uniq:                      # Optimizer._update_count, inlined: hundreds of keys per step
                c = cnt.get(k, begin) + 1
                if k not in synced and k in self._keys:
                    # the update count t of the bias corrections is the OPTIMIZER's (begin_num_update, an
                    # optimizer that has already been stepping elsewhere, states loaded without their
                    # optimizer: optimizer.py:445-462, adam.py:166-175): the engine's count follows it
                    self._set_count(k, c - 1)
                    synced.add(k)
                cnt[k] = c
                if c > top:
                    top = c
            opt_.num_update = top
            self._last_pushed = uniq
            if opt_.param_dict:
                self._sync_mults(uniq)
        self._sync_lr()

    # -- marshalling cache ----------------------------------------------------------------------------
    # A training loop passes the SAME key list and array lists every step (Trainer does); flattening them and
    # building the ctypes arrays again costs more than the engine's replay of its cached launch plan.  An entry
    # is reused only if the very same list objects hold the very same array objects (identity, element by
    # element; the snapshots keep the arrays alive, so an id cannot be recycled).
    @staticmethod
    def _snap(x):
        if isinstance(x, (list, tuple)):
            return tuple(tuple(v) if isinstance(v, (list, tuple)) else v for v in x)
        return x

    @staticmethod
    def _same(x, snap):
        if not isinstance(x, (list, tuple)):
            return x is snap
        if not isinstance(snap, tuple) or len(x) != len(snap):
            return False
        for a, b in zip(x, snap):
            if a is b:
                continue
            if isinstance(a, (list, tuple)) and isinstance(b, tuple) and len(a) == len(b) and all(map(_is, a, b)):
                continue
            return False
        return True

    def _marshalled(self, kind, key, value, out):
        cache = self.__dict__.setdefault("_mcache", {})
        ident = (kind, id(key), id(value), id(out))
        ent = cache.get(ident)
        if ent is not None and self._same(key, ent[0]) and self._same(value, ent[1]) and \
                (out is None or self._same(out, ent[2])):
            return ent[3]
        vkeys, vals, use_str = _ctype_key_value(key, value)
        if out is not None:
            okeys, outs, _ = _ctype_key_value(key, out)
        else:
            okeys, outs = vkeys, vals
        packed = (vkeys, use_str, len(vkeys), _c_keys(vkeys, use_str), _c_vals(vals),
                  len(okeys), _c_keys(okeys, use_str), _c_vals(outs), vals, outs)
        if len(cache) >= 16:
            cache.clear()
        cache[ident] = (self._snap(key), self._snap(value), self._snap(out), packed)
        return packed

    def push(self, key, value, priority=0):
        vkeys, use_str, n, ckeys, cvals, _, _, _, _, _ = self._marshalled(0, key, value, None)
        self._advance_counts(vkeys)
        fn = _LIB.MXKVStorePushEx if use_str else _LIB.MXKVStorePush
        check_call(fn(self.handle, n, ckeys, cvals, ctypes.c_int(priority)))
        self._sync_scalars()

    def pull(self, key, out=None, priority=0, ignore_sparse=True):
        assert out is not None
        keys, vals, use_str = _ctype_key_value(key, out)
        fn = _LIB.MXKVStorePullWithSparseEx if use_str else _LIB.MXKVStorePullWithSparse
        check_call(fn(self.handle, len(keys), _c_keys(keys, use_str), _c_vals(vals), ctypes.c_int(priority),
                      ctypes.c_bool(ignore_sparse)))

    def pushpull(self, key, value, out=None, priority=0):
        vkeys, use_str, n, ckeys, cvals, m, cokeys, couts, _, _ = self._marshalled(1, key, value, out)
        self._advance_counts(vkeys)
        fn = _LIB.MXKVStorePushPullEx if use_str else _LIB.MXKVStorePushPull
        check_call(fn(self.handle, n, ckeys, m, cokeys, cvals, couts, ctypes.c_int(priority)))
        self._sync_scalars()

    def _sync_scalars(self):
        """Nadam's ``m_schedule`` is one product for the whole optimizer, advanced by every fused key update in the
        store: read back after each push, as the update counts are kept in step (``_advance_counts``), so that a
        saved optimizer, a re-sent one and a Python ``step`` taking over all continue from it."""
        if self._fused and getattr(self._optimizer, "fused_name", None) == "nadam":
            self._optimizer.m_schedule = self._get_scalar("m_schedule")

    def _get_scalar(self, name):
        out = ctypes.c_double()
        check_call(_LIB.MXKVB200GetOptimizerScalar(self.handle, c_str(name), ctypes.byref(out)))
        return out.value

    def _set_scalar(self, name, value):
        check_call(_LIB.MXKVB200SetOptimizerScalar(self.handle, c_str(name), ctypes.c_double(value)))

    def broadcast(self, key, value, out, priority=0):
        vkeys, vals, use_str = _ctype_key_value(key, value)
        okeys, outs, _ = _ctype_key_value(key, out)
        fn = _LIB.MXKVStoreBroadcastEx if use_str else _LIB.MXKVStoreBroadcast
        check_call(fn(self.handle, len(vkeys), _c_keys(vkeys, use_str), len(okeys), _c_keys(okeys, use_str),
                      _c_vals(vals), _c_vals(outs), ctypes.c_int(priority)))
        self._keys.update(vkeys)

    def row_sparse_pull(self, key, out=None, priority=0, row_ids=None):
        assert out is not None
        assert row_ids is not None
        if isinstance(row_ids, NDArray):
            row_ids = [row_ids]
        assert isinstance(row_ids, list), "row_ids should be NDArray or list of NDArray"
        first_out = out
        single_rowid = False
        if len(row_ids) == 1 and isinstance(out, list):
            single_rowid = True
            first_out = [out[0]]
        keys, vals, use_str = _ctype_key_value(key, first_out)
        _, rids, _ = _ctype_key_value(key, row_ids)
        assert len(rids) == len(vals), "the number of row_ids doesn't match the number of values"
        fn = _LIB.MXKVStorePullRowSparseEx if use_str else _LIB.MXKVStorePullRowSparse
        check_call(fn(self.handle, len(keys), _c_keys(keys, use_str), _c_vals(vals), _c_vals(rids),
                      ctypes.c_int(priority)))
        if single_rowid:
            for out_i in out[1:]:
                out[0].copyto(out_i)

    # -- capabilities / metadata -------------------------------------------------
    @staticmethod
    def is_capable(capability):
        if capability.lower() == KVStoreBase.OPTIMIZER:
            return True
        raise MXNetError("Unknown capability: {}".format(capability))

    @property
    def type(self):
        t = ctypes.c_char_p()
        check_call(_LIB.MXKVStoreGetType(self.handle, ctypes.byref(t)))
        return t.value.decode()

    @property
    def rank(self):
        r = ctypes.c_int()
        check_call(_LIB.MXKVStoreGetRank(self.handle, ctypes.byref(r)))
        return r.value

    @property
    def num_workers(self):
        r = ctypes.c_int()
        check_call(_LIB.MXKVStoreGetGroupSize(self.handle, ctypes.byref(r)))
        return r.value

    def set_deferred(self, on=True):
        """Queue push / pushpull calls and issue them at the next flush point in priority order, merged
        (MXKVB200SetDeferred): the engine-side meaning of ``priority``."""
        check_call(_LIB.MXKVB200SetDeferred(self.handle, 1 if on else 0))

    def flush(self):
        check_call(_LIB.MXKVB200Flush(self.handle))

    def deferred_batches(self):
        n = ctypes.c_int64()
        check_call(_LIB.MXKVB200GetDeferredBatches(self.handle, ctypes.byref(n)))
        return n.value

    def plan_hits(self):
        """push / pushpull calls served from a cached launch plan (MXKVB200GetPlanHits)"""
        n = ctypes.c_int64()
        check_call(_LIB.MXKVB200GetPlanHits(self.handle, ctypes.byref(n)))
        return n.value

    def set_gradient_compression(self, compression_params):
        """kvstore.py:505-557: 'device' and 'dist' stores only"""
        if not (("device" in self.type) or ("dist" in self.type)):
            raise Exception("Gradient compression is not supported for this type of kvstore")
        keys = list(compression_params.keys())
        vals = [str(compression_params[k]) for k in keys]
        check_call(_LIB.MXKVStoreSetGradientCompression(self.handle, len(keys), c_str_array(keys),
                                                        c_str_array(vals)))

    def _barrier(self):
        check_call(_LIB.MXKVStoreBarrier(self.handle))

    # -- optimizer ---------------------------------------------------------------------
    def set_optimizer(self, optimizer):
        """Recognised optimizers run fused inside the reduce kernel; anything else goes through
        the Python updater callback like the reference (kvstore.py:559-606)."""
        fresh = optimizer is not self._optimizer          # a new optimizer object: new (empty) state, as in the reference
        self._optimizer = optimizer
        self._synced = set()
        if opt.fused_name_of(optimizer):
            if self._updater is not None:
                # the reference's set_optimizer always REPLACES the updater (kvstore.py:559-606): a callback
                # left over from an earlier optimizer must not keep running
                check_call(_LIB.MXKVStoreSetUpdaterEx(self.handle, None, None, None))
                self._updater = None
            kw = optimizer.fused_kwargs()
            if fresh:
                kw["reset_states"] = True
            keys = list(kw.keys())
            vals = [str(kw[k]) for k in keys]
            check_call(_LIB.MXKVB200SetOptimizer(self.handle, c_str(optimizer.fused_name), len(keys),
                                                 c_str_array(keys), c_str_array(vals)))
            self._fused = True
            self._last_lr = optimizer.learning_rate
            now = optimizer.key_multipliers()
            for k in [k for k in self._mults if k not in now and self._mults[k] != (1.0, 1.0)]:
                self.set_mult(k, 1.0, 1.0)              # a multiplier of the previous optimizer
            for k, (lm, wm) in now.items():
                self.set_mult(k, lm, wm)
            if hasattr(optimizer, "no_trust_ratio_indices"):
                for k in optimizer.no_trust_ratio_indices():
                    self.set_key_flag(k, "no_trust_ratio", 1)
        else:
            self._fused = False
            self._set_updater(opt.get_updater(optimizer, native=False))

    def _set_count(self, key, count):
        if isinstance(key, str):
            check_call(_LIB.MXKVB200SetUpdateCount(self.handle, 0, c_str(key), ctypes.c_int64(count)))
        else:
            check_call(_LIB.MXKVB200SetUpdateCount(self.handle, int(key), None, ctypes.c_int64(count)))

    def _sync_mults(self, keys):
        """``Parameter.lr_mult`` / ``wd_mult`` are read at every update by the reference
        (optimizer.py:479-487,518-525 through ``param_dict``), so a change between steps takes effect at once
        (tests/python/unittest/test_gluon_trainer.py:94-100,131-149): the engine's per-key multipliers follow."""
        opt_ = self._optimizer
        if not (self._fused and opt_ is not None and opt_.param_dict):
            return
        pd, seen = opt_.param_dict, self._mults
        for k in keys:
            if k in pd:
                m = (opt_._mult(opt_.lr_mult, "lr_mult", k), opt_._mult(opt_.wd_mult, "wd_mult", k))
                if seen.get(k, (1.0, 1.0)) != m:
                    self.set_mult(k, m[0], m[1])

    def set_mult(self, key, lr_mult=1.0, wd_mult=1.0):
        self._mults[key] = (lr_mult, wd_mult)
        if isinstance(key, str):
            check_call(_LIB.MXKVB200SetOptimizerMult(self.handle, 0, c_str(key), ctypes.c_float(lr_mult),
                                                     ctypes.c_float(wd_mult)))
        else:
            check_call(_LIB.MXKVB200SetOptimizerMult(self.handle, int(key), None, ctypes.c_float(lr_mult),
                                                     ctypes.c_float(wd_mult)))

    def set_key_flag(self, key, name, value=1):
        """Per-key switch of a fused optimizer (MXKVB200SetKeyFlag)."""
        if isinstance(key, str):
            check_call(_LIB.MXKVB200SetKeyFlag(self.handle, 0, c_str(key), c_str(name), int(value)))
        else:
            check_call(_LIB.MXKVB200SetKeyFlag(self.handle, int(key), None, c_str(name), int(value)))

    def overflow(self):
        """True if the last push (optimizer created with ``skip_nonfinite=True``) met a non-finite
        gradient and therefore changed nothing; waits for the push to finish and clears the flag."""
        out = ctypes.c_int(0)
        check_call(_LIB.MXKVB200GetOverflow(self.handle, ctypes.byref(out)))
        if out.value and self._optimizer is not None:
            # the skipped step does not count on the Python side either
            cnt = self._optimizer._index_update_count
            for k in getattr(self, "_last_pushed", []):
                if cnt.get(k, 0) > self._optimizer.begin_num_update:
                    cnt[k] -= 1
            self._optimizer.num_update = max([self._optimizer.begin_num_update] + list(cnt.values()))
        return bool(out.value)

    def _send_command_to_servers(self, head, body):
        """kvstore.py:714-729; a no-op for single-node stores (include/mxnet/kvstore.h:432)."""
        check_call(_LIB.MXKVStoreSendCommmandToServers(self.handle, ctypes.c_int(head), c_str(body)))

    def _sync_lr(self):
        if self._fused and self._optimizer is not None:
            lr = self._optimizer.learning_rate
            if lr != self._last_lr:
                check_call(_LIB.MXKVB200SetLearningRate(self.handle, ctypes.c_double(lr)))
                self._last_lr = lr

    def _set_updater(self, updater):
        """kvstore.py:674-712: int- and str-key ctypes trampolines; the callee frees the handles."""
        self._updater = updater

        def _wrap(key, recv_h, local_h, _):
            recv = NDArray(ctypes.c_void_p(recv_h))
            local = NDArray(ctypes.c_void_p(local_h))
            if isinstance(key, bytes):
                key = key.decode()
            updater(key, recv, local)

        proto = ctypes.CFUNCTYPE(None, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)
        sproto = ctypes.CFUNCTYPE(None, ctypes.c_char_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p)
        self._updater_func = proto(_wrap)
        self._str_updater_func = sproto(_wrap)
        check_call(_LIB.MXKVStoreSetUpdaterEx(self.handle, self._updater_func, self._str_updater_func, None))

    def _state_handle(self, key, which):
        out = ctypes.c_void_p()
        if isinstance(key, str):
            check_call(_LIB.MXKVB200GetState(self.handle, 0, c_str(key), which, ctypes.byref(out)))
        else:
            check_call(_LIB.MXKVB200GetState(self.handle, int(key), None, which, ctypes.byref(out)))
        return NDArray(out) if out.value else None

    def save_optimizer_states(self, fname, dump_optimizer=False):
        """Same file role as kvstore.py:647-660 (pickle of {key: states}); for the fused path the
        states are read back from engine memory (sharded states are gathered first)."""
        if not self._fused:
            assert self._updater is not None, "Cannot save states for distributed training"
            with open(fname, "wb") as fout:
                fout.write(self._updater.get_states(dump_optimizer))
            return
        with open(fname, "wb") as fout:
            fout.write(self._dump_fused_states(dump_optimizer))

    def _dump_fused_states(self, dump_optimizer=False):
        states = {}
        for k in sorted(self._keys, key=str):
            ent = {}
            for which, name in ((1, "weight32"), (2, "state0"), (3, "state1"), (4, "state2")):
                h = self._state_handle(k, which)
                if h is not None:
                    ent[name] = h.asnumpy()
            cnt = ctypes.c_int64()
            if isinstance(k, str):
                check_call(_LIB.MXKVB200GetUpdateCount(self.handle, 0, c_str(k), ctypes.byref(cnt)))
            else:
                check_call(_LIB.MXKVB200GetUpdateCount(self.handle, int(k), None, ctypes.byref(cnt)))
            ent["count"] = cnt.value
            states[k] = ent
        payload = {"format": "mxkv_b200_fused_v1", "states": states}
        if dump_optimizer:
            payload["optimizer"] = self._optimizer
        return pickle.dumps(payload)

    def load_optimizer_states(self, fname):
        with open(fname, "rb") as fin:
            blob = fin.read()
        if not self._fused:
            assert self._updater is not None, "Cannot load states for distributed training"
            self._updater.set_states(blob)
            return
        payload = pickle.loads(blob)
        if payload.get("optimizer") is not None:
            # updater.py:118-127: a dumped optimizer replaces the current one (its update counts and learning
            # rate included); the engine's arrays are untouched by set_optimizer
            self.set_optimizer(payload["optimizer"])
        self._load_fused_states(payload)

    def _load_fused_states(self, blob, only=None):
        payload = pickle.loads(blob) if isinstance(blob, bytes) else blob
        assert payload.get("format") == "mxkv_b200_fused_v1", "not a fused-optimizer state file"
        for k, ent in payload["states"].items():
            if only is not None and k not in only:
                continue
            for which, name in ((1, "weight32"), (2, "state0"), (3, "state1"), (4, "state2")):
                if name in ent:
                    v = _nd.array(ent[name], dtype=np.float32)
                    if isinstance(k, str):
                        check_call(_LIB.MXKVB200SetState(self.handle, 0, c_str(k), which, v.handle))
                    else:
                        check_call(_LIB.MXKVB200SetState(self.handle, int(k), None, which, v.handle))
            self._set_count(k, ent["count"])
        # whatever the file says, the next update counts from the current optimizer's table (updater.py:118-127
        # restores the optimizer only when it was dumped along)
        self._synced -= set(payload["states"])
        _nd.waitall()


@KVStoreBase.register
class B200Device(KVStore):
    """``create('b200device')`` -- the name under which the engine registers itself in a
    KVStoreBase registry (see INTEGRATION.md for registering it as 'device' in the reference)."""

    def __init__(self):
        super(B200Device, self).__init__("device")


def create(name="local"):
    """Creates a new KVStore (base.py:406-461): registry first, native store otherwise."""
    if not isinstance(name, str):
        raise TypeError("name must be a string")
    lname = name.lower()
    if lname in KVStoreBase.kv_registry:
        return KVStoreBase.kv_registry[lname]()
    return KVStore(name)


def fence(dev_id=None):
    """Make the caller's CUDA stream(s) wait for everything the engine has queued (async)."""
    from .context import num_gpus
    devs = range(num_gpus()) if dev_id is None else [dev_id]
    for d in devs:
        check_call(_LIB.MXKVB200Fence(ctypes.c_int(d)))


def set_auto_fence(flag):
    check_call(_LIB.MXKVB200SetAutoFence(ctypes.c_int(1 if flag else 0)))


VARIANTS = {"per_thread": 0, "bulk": 1, "nvls": 2, "tree": 3}


def launch_count(variant=None):
    """Kernels launched by the engine so far; with ``variant`` ('per_thread' | 'bulk' | 'nvls' | 'tree') the dense
    reduce(+update) launches of that kernel variant only."""
    n = ctypes.c_int64()
    if variant is None:
        check_call(_LIB.MXKVB200GetLaunchCount(ctypes.byref(n)))
    else:
        check_call(_LIB.MXKVB200GetVariantLaunchCount(VARIANTS.get(variant, variant), ctypes.byref(n)))
    return n.value


def set_tuning(chunk_elems=0, threads=0, max_blocks=-1, bulk=-1):
    """MXKVB200SetTuning: chunk_elems / threads 0 keep the current value, max_blocks <= 0 = resident capacity.  ``bulk``: 0 never the staged kernel, 1 auto, 2 always
    where eligible (float32, 16-byte aligned, sizes that are multiples of 4)."""
    check_call(_LIB.MXKVB200SetTuning(ctypes.c_int64(chunk_elems), int(threads), int(max_blocks), int(bulk)))


def set_nvls_tuning(unroll=0, pipe=-1, grid=-1, threads=0):
    """MXKVB200SetNvlsTuning (same values on every rank)."""
    check_call(_LIB.MXKVB200SetNvlsTuning(int(unroll), int(pipe), int(grid), int(threads)))


def set_nvls(mode):
    """MXKVB200SetNvls: 0 never, 1 auto (above 4 ranks), 2 whenever the arrays have a multicast alias."""
    check_call(_LIB.MXKVB200SetNvls(int(mode)))
