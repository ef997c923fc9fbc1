"""What one GPU can stream for three fp32 reads and three fp32 writes per element: the access pattern of a fused
SGD-momentum pushpull at N = 1 (g, w, mom in; stored w, mom, out), which is what bench.py's headline measures.

The kernels (tools/hbm_stream.cu, compiled here into a temporary directory) compute x = a + b, y = b + c, z = a + c
over six arrays of --elements floats (default 2^26: 256 MB each, far beyond the 50 MB L2):

  staged      the staged dense kernel's scheme: cp.async.bulk of the three inputs into an mbarrier ring in shared
              memory, 256 threads, two blocks per SM; at several tile x stage points, each with the stage released
              after the stores (as the staged kernel did) and before them (operands copied to registers first)
  plain       per-thread ld.v4 / st.v4 grid-stride loops with 1, 2 and 4 packets of each input in flight
  read/write  three reads only, three writes only, for context

Rates are bytes the kernel must move (24 per element for the 3R/3W kernels, 12 for read / write only) over the median
kernel time from CUDA events, over --reps launches per round and --rounds rounds.  The card's name, power limit and
SM clock are read with nvidia-smi in the same call.  The best 3R/3W rate is the stream ceiling the staged kernel is
measured against (profiles/README.md).

    python tools/hbm_stream.py [--elements 67108864] [--reps 20] [--rounds 3] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))

STAGED_POINTS = [(1024, 4), (2048, 2), (2048, 3), (2048, 4), (4096, 2)]
PLAIN_UNROLLS = [1, 2, 4]


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, check=True).stdout
    name, power, max_clock, clock = [x.strip() for x in out.strip().splitlines()[0].split(",")]
    return {"name": name, "power_limit": power, "max_sm_clock": max_clock, "sm_clock_sampled": clock}


def compile_lib(tmp):
    nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    so = os.path.join(tmp, "libhbm_stream.so")
    subprocess.check_call([nvcc, "-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-shared",
                           "-Xcompiler", "-fPIC", "-o", so, os.path.join(HERE, "hbm_stream.cu")])
    lib = ctypes.CDLL(so)
    p, i, ll = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong
    lib.hs_staged.argtypes = [p, p, p, p, p, p, ll, i, i, i, i, p]
    lib.hs_plain.argtypes = [p, p, p, p, p, p, ll, i, i, p]
    lib.hs_read.argtypes = [p, p, p, p, ll, i, p]
    lib.hs_write.argtypes = [p, p, p, ll, i, p]
    lib.hs_staged_occupancy.argtypes = [i, i, i]
    return lib


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--elements", type=int, default=1 << 26)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a GPU"
    n = args.elements - args.elements % 4096
    info = card()
    with tempfile.TemporaryDirectory() as tmp:
        lib = compile_lib(tmp)
        dev = torch.device("cuda", 0)
        sms = torch.cuda.get_device_properties(dev).multi_processor_count
        ins = [torch.rand(n, device=dev) for _ in range(3)]
        outs = [torch.empty(n, device=dev) for _ in range(3)]
        sink = torch.zeros(4, device=dev)
        a, b, c = (t.data_ptr() for t in ins)
        x, y, z = (t.data_ptr() for t in outs)
        stream = torch.cuda.current_stream(dev)
        sp = stream.cuda_stream

        cases = []
        for tile, st in STAGED_POINTS:
            for early in (0, 1):
                occ = lib.hs_staged_occupancy(early, tile, st)
                if occ < 1:
                    continue
                cases.append(("staged %d x %d %s" % (tile, st, "release-before-stores" if early else "release-after-stores"),
                              24, (lambda tile=tile, st=st, early=early, occ=occ:
                                   lib.hs_staged(a, b, c, x, y, z, n, tile, st, early, occ * sms, sp)),
                              {"tile": tile, "stages": st, "release_before_stores": bool(early), "blocks_per_sm": occ}))
        for u in PLAIN_UNROLLS:
            cases.append(("plain ld.v4/st.v4, %d packet(s) in flight" % u, 24,
                          (lambda u=u: lib.hs_plain(a, b, c, x, y, z, n, u, sms * 8, sp)), {"unroll": u}))
        cases.append(("read only (3 reads)", 12, lambda: lib.hs_read(a, b, c, sink.data_ptr(), n, sms * 8, sp), {}))
        cases.append(("write only (3 writes)", 12, lambda: lib.hs_write(x, y, z, n, sms * 8, sp), {}))

        ref = [ins[0] + ins[1], ins[1] + ins[2], ins[0] + ins[2]]
        times = {name: [] for name, _, _, _ in cases}
        wrong = set()
        for _ in range(args.rounds):                 # the cases alternate within a round: the machine is shared
            for name, _, fn, _ in cases:
                for _ in range(3):
                    assert fn() == 0, name
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                       for _ in range(args.reps)]
                for e0, e1 in evs:
                    e0.record(stream)
                    fn()
                    e1.record(stream)
                torch.cuda.synchronize()
                times[name].append(statistics.median(e0.elapsed_time(e1) for e0, e1 in evs))
                if "read only" not in name and "write only" not in name:
                    if not all(torch.equal(o, r) for o, r in zip(outs, ref)):
                        wrong.add(name)
                    for o in outs:
                        o.zero_()
        result = {"card": info, "elements": n, "reps": args.reps, "rounds": args.rounds, "cases": []}
        for name, bpe, _, meta in cases:
            ms = statistics.median(times[name])
            ent = dict(meta, case=name, ms=ms, ms_rounds=times[name], gbs=n * bpe / (ms * 1e-3) / 1e9,
                       results_correct=name not in wrong)
            result["cases"].append(ent)
            print("%-52s %8.1f us  %7.0f GB/s%s" % (name, ms * 1e3, ent["gbs"], "" if ent["results_correct"] else
                                                     "  WRONG RESULTS"), flush=True)
        # a kernel that computed wrong results does not count towards the ceiling
        best = max((e for e in result["cases"] if "only" not in e["case"] and e["results_correct"]),
                   key=lambda e: e["gbs"])
        result["r_star_gbs"] = best["gbs"]
        result["r_star_case"] = best["case"]
        result["card"]["sm_clock_after"] = card()["sm_clock_sampled"]
    print("R* (best 3R/3W): %.0f GB/s, %s" % (best["gbs"], best["case"]))
    print("card: %s, power limit %s, max SM clock %s, SM clock sampled %s / %s" % (
        info["name"], info["power_limit"], info["max_sm_clock"], info["sm_clock_sampled"], result["card"]["sm_clock_after"]))
    line = json.dumps(result)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    sys.exit(main())
