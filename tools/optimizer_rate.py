"""Step time of the fused NAG against fused SGD-momentum at N = 1 (one GPU, one gradient per key), and of NAG through
the Python `step` (use_fused_step=False, the only way to run NAG before the fused kernel existed).  With
`--pair adabelief`: the fused AdaBelief against the fused Adam instead (both read g, w, mean, var and write stored w,
mean, var, out: 32 bytes per float32 element).  With `--pair rmsprop`: the fused RMSProp against the fused SGD-momentum
(24 bytes per float32 element each), the fused centered RMSProp against the fused Adam (40 against 32 bytes: it reads
g, w, mean, var, mom and writes stored w, mean, var, mom, out), and RMSProp through the Python `step`.  With
`--pair signum`: the fused Signum against the fused SGD-momentum (24 bytes per float32 element each), the fused
signSGD against the fused SGD (16 bytes each: read g, w; write stored w, out), and Signum through the Python `step`.
With `--pair ftml`: the fused FTML against the fused centered RMSProp (40 bytes per float32 element each: read g, w
and three states; write stored w, three states, out), and FTML through the Python `step`.  With `--pair adamax` /
`--pair adadelta`: the fused Adamax / AdaDelta against the fused Adam (32 bytes per float32 element each: read g, w,
s0, s1; write stored w, s0, s1, out), and the optimizer through the Python `step`.  With `--pair nadam`: the fused
Nadam against the fused Adam (the same 32 bytes per element; Nadam's per-key schedule scalars ride along with the work
list), and Nadam through the Python `step`.

Two key sets: the bench sweep (9 float32 keys, 2^10 ... 2^26 elements) and ResNet-50's 193 gradient-carrying arrays
(bench.py: keyset).  Both fused optimizers move the same bytes per element (read g, w, mom; write stored w, mom, out),
so they are timed alternately in one process, `--rounds` times each.  Per case: ms per step from CUDA events on the
engine's stream (the Python path: host clock around a device synchronise, its torch ops run on torch's stream), the
dense kernel variant that ran (launch counters), and one step checked against the CPU oracle.  The card's name and
power limit are read with nvidia-smi in the same call and printed with the numbers.

    python tools/optimizer_rate.py [--pair nag|adabelief|rmsprop|signum|ftml|adamax|adadelta|nadam] [--steps 200] [--warmup 20] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import keyset, nelem, tile_fill  # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))

KW = dict(learning_rate=0.01, momentum=0.9, wd=1e-4)
KW_ADAPTIVE = dict(learning_rate=0.001, wd=1e-4)
KW_FTML = dict(learning_rate=0.0025, wd=1e-4)
KW_STEP = {"adamax": dict(learning_rate=0.002, wd=1e-4), "adadelta": dict(learning_rate=1.0, wd=1e-4),
           "nadam": dict(learning_rate=0.001, wd=1e-4)}
# --pair: (baseline, optimizer under test) pairs, alternated in one process; the python step is timed for the first
# optimizer under test where it was the only way to run it (NAG, RMSProp, Signum, FTML, Adamax, AdaDelta, Nadam)
PAIRS = {"nag": [("sgd", "nag")], "adabelief": [("adam", "adabelief")],
         "rmsprop": [("sgd", "rmsprop"), ("adam", "rmsprop_centered")],
         "signum": [("sgd", "signum"), ("sgd_plain", "signsgd")],
         "ftml": [("rmsprop_centered", "ftml")], "adamax": [("adam", "adamax")], "adadelta": [("adam", "adadelta")],
         "nadam": [("adam", "nadam")]}
PYTHON_STEP = ("nag", "rmsprop", "signum", "ftml", "adamax", "adadelta", "nadam")
LABELS = {"sgd": "sgd_momentum", "nag": "nag", "adam": "adam", "adabelief": "adabelief", "rmsprop": "rmsprop",
          "rmsprop_centered": "rmsprop (centered)", "sgd_plain": "sgd", "signum": "signum",
          "signsgd": "signum (momentum 0: signsgd)", "ftml": "ftml",
          "adamax": "adamax", "adadelta": "adadelta", "nadam": "nadam"}
VARIANTS = ("per_thread", "bulk", "nvls", "tree")


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = [x.strip() for x in out.split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def engine_stream(mx, torch):
    from mxnet_b200.base import _LIB, check_call
    sp = ctypes.c_void_p()
    check_call(_LIB.MXKVB200GetEngineStream(0, ctypes.byref(sp)))
    return torch.cuda.ExternalStream(sp.value, device=torch.device("cuda", 0))


class Case(object):
    def __init__(self, mx, shapes, optname, fused):
        self.mx, self.shapes, self.optname, self.fused = mx, shapes, optname, fused
        self.keys = list(range(len(shapes)))
        w0 = [tile_fill(np.random.default_rng(99), 0, 1, s) for s in shapes]
        self.w0 = w0
        self.grads_np = [tile_fill(np.random.default_rng(1234 + k), -1, 1, s) for k, s in enumerate(shapes)]
        self.kv = mx.kv.create("device")
        self.kv.init(self.keys, [mx.nd.array(w, mx.gpu(0)) for w in w0])
        self.kw = KW if optname in ("sgd", "nag", "signum") else KW_ADAPTIVE
        if optname.startswith("rmsprop"):
            self.kw = dict(KW_ADAPTIVE, centered=optname == "rmsprop_centered")
        if optname in ("sgd_plain", "signsgd"):
            self.kw = dict(KW, momentum=0.0)
        if optname == "ftml":
            self.kw = KW_FTML
        if optname in KW_STEP:
            self.kw = KW_STEP[optname]
        cls = {"sgd": mx.optimizer.SGD, "nag": mx.optimizer.NAG, "adam": mx.optimizer.Adam,
               "adabelief": mx.optimizer.AdaBelief, "rmsprop": mx.optimizer.RMSProp,
               "rmsprop_centered": mx.optimizer.RMSProp, "sgd_plain": mx.optimizer.SGD, "signum": mx.optimizer.Signum,
               "signsgd": mx.optimizer.Signum, "ftml": mx.optimizer.FTML,
               "adamax": mx.optimizer.Adamax, "adadelta": mx.optimizer.AdaDelta, "nadam": mx.optimizer.Nadam}[optname]
        opt = cls(**dict(self.kw, **({} if fused else {"use_fused_step": False})))
        self.kv.set_optimizer(opt)
        self.grads = [mx.nd.array(g, mx.gpu(0)) for g in self.grads_np]
        self.outs = [mx.nd.empty(s, mx.gpu(0)) for s in shapes]

    def step(self):
        self.kv.pushpull(self.keys, self.grads, out=self.outs)

    def check(self):
        """the first step against the oracle: bits for the fused kernels, the reference's test_nag tolerance for the
        Python step"""
        from oracle import oracle as O
        self.step()
        self.mx.nd.waitall()
        import torch
        torch.cuda.synchronize()
        if self.optname == "nag":
            import nag_oracle as N
            oopt = N.OracleNAG(**self.kw)
        elif self.optname == "adabelief":
            import adabelief_oracle as A
            oopt = A.OracleAdaBelief(**self.kw)
        elif self.optname.startswith("rmsprop"):
            import rmsprop_oracle as R
            oopt = R.OracleRMSProp(**self.kw)
        elif self.optname in ("signum", "signsgd"):
            import signum_oracle as S
            oopt = S.OracleSignum(**self.kw)
        elif self.optname == "ftml":
            import ftml_oracle as F
            oopt = F.OracleFTML(**self.kw)
        elif self.optname == "adamax":
            import adamax_oracle as AM
            oopt = AM.OracleAdamax(**self.kw)
        elif self.optname == "adadelta":
            import adadelta_oracle as AD
            oopt = AD.OracleAdaDelta(**self.kw)
        elif self.optname == "nadam":
            import nadam_oracle as NA
            oopt = NA.OracleNadam(**self.kw)
        else:
            oopt = O.OracleOptimizer("sgd" if self.optname == "sgd_plain" else self.optname, **self.kw)
        exact, close = True, True
        for k in self.keys:
            w = self.w0[k].reshape(-1).copy()
            oopt.update(k, w, self.grads_np[k].reshape(-1))
            got = self.outs[k].asnumpy().reshape(-1)
            exact = exact and np.array_equal(got.view(np.uint32), w.view(np.uint32))
            close = close and bool(np.allclose(got, w, rtol=1e-3, atol=1e-4))
        return "bit-exact" if exact else ("within rtol 1e-3 / atol 1e-4" if close and not self.fused else "FAILED")


def time_case(mx, torch, stream, case, steps, warmup):
    for _ in range(warmup):
        case.step()
    mx.nd.waitall()
    torch.cuda.synchronize()
    before = {v: mx.kv.launch_count(v) for v in VARIANTS}
    if case.fused:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(steps):
            case.step()
        e1.record(stream)
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / steps
    else:
        t0 = time.perf_counter()
        for _ in range(steps):
            case.step()
        mx.nd.waitall()
        torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3 / steps
    now = {v: mx.kv.launch_count(v) for v in VARIANTS}
    used = [v for v in VARIANTS if now[v] > before[v]]
    return ms, "+".join(used) if used else "python"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--pair", choices=sorted(PAIRS), default="nag")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    import mxnet_b200 as mx
    info = card()
    stream = engine_stream(mx, torch)
    result = {"card": info, "pair": args.pair, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds,
              "cases": []}
    pairs = PAIRS[args.pair]
    for ksname in ("sweep", "resnet50"):
        shapes = keyset(ksname)
        cases = [(o, True) for pair in pairs for o in pair]
        if ksname == "resnet50" and pairs[0][1] in PYTHON_STEP:
            cases.append((pairs[0][1], False))
        built = {c: Case(mx, shapes, c[0], c[1]) for c in cases}
        checks = {c: built[c].check() for c in cases}
        times = {c: [] for c in cases}
        variants = {}
        for _ in range(args.rounds):                 # alternate the cases: the machine is shared
            for c in cases:
                ms, variants[c] = time_case(mx, torch, stream, built[c], args.steps, args.warmup)
                times[c].append(ms)
        for c in cases:
            ent = {"keyset": ksname, "keys": len(shapes), "elements": int(sum(nelem(s) for s in shapes)),
                   "optimizer": LABELS[c[0]] + ("" if c[1] else " (python step)"),
                   "ms_per_step": times[c], "ms_median": float(np.median(times[c])), "variant": variants[c],
                   "oracle_check": checks[c]}
            result["cases"].append(ent)
            print("%-8s %-28s %8.3f ms/step (runs %s)  variant %-10s oracle %s" % (
                ksname, ent["optimizer"], ent["ms_median"], ", ".join("%.3f" % t for t in times[c]), variants[c],
                checks[c]), flush=True)
        del built
        mx.nd.waitall()
    print("card: %s, power limit %s, max SM clock %s" % (info["name"], info["power_limit"], info["max_sm_clock"]))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
