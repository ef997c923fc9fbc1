"""The engine's host logic exercised on a simulated CUDA runtime (tests/sim): the `-m gpu` parity tests run,
unchanged, against the product's own object files re-linked to a stand-in libcudart whose kernel launches are
carried out by semantic emulators built from the kernels' arithmetic headers.  Everything around the kernels
is real: C ABI, key bookkeeping, placement over several (simulated) GPUs, replica / optimizer-state / shard
management, work lists, aliasing rules, launch sequences.  See tests/sim/README.md for what this can and
cannot establish."""
import importlib.util
import os
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIM = os.path.join(ROOT, "tests", "sim")


@pytest.fixture(scope="module")
def sim_lib():
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("needs g++ and nvcc to build the simulated runtime")
    spec = importlib.util.spec_from_file_location("build_sim", os.path.join(SIM, "build_sim.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    lib, _ = b.build()
    return lib


def _workers():
    """the inner runs are hundreds of independent small tests: spread them over a few processes (each has its own
    simulated GPUs) when pytest-xdist is there"""
    try:
        import xdist  # noqa: F401
    except ImportError:
        return []
    return ["-n", str(max(1, min(4, (os.cpu_count() or 2) // 2)))]


def _run(sim_lib, devices, files, extra=()):
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES=str(devices))
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider"] + _workers() + list(extra) + \
          [os.path.join(ROOT, "tests", f) for f in files]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    if r.returncode != 0:
        # keep everything (a crash report's traceback sits ABOVE its long list of extension modules)
        log = os.path.join(SIM, "_build", "last_failure_%d_devices.log" % devices)
        with open(log, "w") as f:
            f.write(r.stdout + "\n==== stderr ====\n" + r.stderr)
        cut = r.stderr.find("Extension modules:")
        err = r.stderr[:cut] if cut >= 0 else r.stderr
        assert False, "exit code %d (full output in %s)\n%s\n%s" % (r.returncode, log, r.stdout[-1500:], err[-3000:])
    return r.stdout


def _passed(out):
    import re
    m = re.search(r"(\d+) passed", out)
    return int(m.group(1)) if m else 0


def test_single_gpu_paths(sim_lib):
    out = _run(sim_lib, 1, ["test_gpu_dense.py", "test_gpu_reference_kats.py", "test_gpu_rsp.py",
                            "test_gpu_norm_opt.py", "test_gpu_compression.py", "test_gpu_updater.py",
                            "test_gpu_y_trainer_nd.py", "test_gpu_y_semantics.py", "test_gpu_zz_threads.py",
                            "test_gpu_lowp_optimizers.py", "test_gpu_rsp_edges.py", "test_gpu_norm_edges.py",
                            "test_gpu_compression_edges.py"])
    assert _passed(out) >= 100, out[-500:]


@pytest.mark.parametrize("devices", [2, 4, 8])
def test_single_process_multi_gpu_paths(sim_lib, devices):
    """one-shot and two-shot (sharded) exchange, sharded optimizer state, layer-wise optimizers with norms added
    across the shards, compression, the updater callback -- over 2, 4 and 8 simulated GPUs."""
    out = _run(sim_lib, devices, ["test_gpu_multi.py", "test_gpu_compression.py", "test_gpu_rsp.py",
                                  "test_gpu_y_placement.py", "test_gpu_y_trainer_nd.py", "test_gpu_y_semantics.py", "test_gpu_zz_threads.py",
                                  "test_gpu_zzz_tree.py",
                                  "test_gpu_lowp_optimizers.py::test_multi_gpu_sharded_master_and_state_with_a_checkpoint",
                                  "test_gpu_rsp_edges.py::test_multi_gpu_localise_phase",
                                  "test_gpu_norm_edges.py::test_sharded_key_with_small_chunks",
                                  "test_gpu_compression_edges.py::test_several_consumers_and_a_moving_slot"],
               extra=["-k", "not one_process_per_gpu"])
    assert _passed(out) >= 30, out[-500:]


def test_host_code_under_address_and_ub_sanitizers():
    """The engine's host code (and the stand-in runtime) rebuilt with AddressSanitizer + UBSan, driven through
    the placement random walks, the multi-GPU parity tests and the row_sparse paths on 4 simulated GPUs: replica
    vectors that reallocate while pointers into them are held, work lists, state migration, C-ABI buffers.  Any
    report aborts the run.  (The reference's counterpart is its USE_ASAN CI job, CMakeLists.txt:88.)"""
    if shutil.which("g++") is None or not os.path.exists("/usr/local/cuda/bin/nvcc"):
        pytest.skip("needs g++ and nvcc")
    spec = importlib.util.spec_from_file_location("build_sim", os.path.join(SIM, "build_sim.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    san = b.sanitizer_env()
    if not all(os.path.isabs(x) and os.path.exists(x) for x in san["LD_PRELOAD"].split(":")):
        pytest.skip("libasan / libubsan not installed")
    lib, _ = b.build_sanitized()
    env = dict(os.environ)
    env.update(san)
    # (user-level contexts switch stacks behind the sanitizer's back: the dense and tree kernels run from source on
    # the OS-thread engine here -- which also makes a block's threads truly concurrent --, the layer-wise-optimizer and
    # row_sparse kernels, which need their real thread counts, take the independent emulators)
    env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=lib, MXKV_SIM_DEVICES="4", MXKV_SIM_ENGINE="threads",
               MXKV_SIM_NORM="semantic", MXKV_SIM_RSP="semantic")
    cmd = [sys.executable, "-m", "pytest", "-q", "-m", "gpu", "-p", "no:cacheprovider", "-x",
           "-k", "not one_process_per_gpu"] + _workers() + \
          [os.path.join(ROOT, "tests", f) for f in ("test_gpu_y_placement.py", "test_gpu_multi.py", "test_gpu_rsp.py",
                                                    "test_gpu_updater.py", "test_gpu_zzz_tree.py")]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=1500)
    tail = (r.stdout + r.stderr)[-4000:]
    assert r.returncode == 0, tail
    assert "AddressSanitizer" not in tail and "runtime error" not in tail, tail
    assert _passed(r.stdout) >= 100, tail


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_process_per_gpu_on_simulator(sim_lib, world, tmp_path):
    """The torchrun deployment shape without GPUs: `world` processes, each with one simulated GPU, peer memory
    over POSIX shared memory (the stand-in for CUDA IPC), the real flag rendezvous between the emulated kernels,
    files as the bootstrap process group.  Runs every scenario of tests/mp_worker.py except the torch-tensor
    and NVSwitch-multicast ones."""
    import glob
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world))
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_worker.py")], env=e, cwd=ROOT,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=900)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:                       # in case a worker died before its exit handler ran
            for f in glob.glob("/dev/shm/mxkvsim_%d_*" % p.pid):
                os.unlink(f)
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, out[-3000:])
        assert "MP_WORKER_OK rank %d" % r in out, out[-2000:]


def test_layerwise_kernels_from_source_match_the_emulators_bit_for_bit(sim_lib):
    """csrc/norm_kernels.cu run from its own source -- 512-thread blocks as user-level contexts, __shfl_xor_sync as a
    lane exchange -- against the emulators of tests/sim/sim_kernels.cc, which restate the hardware's summation order
    (thread-strided partials, xor tree inside a warp, warps in order): LAMB / LANS / LARS over 1 ... 3 simulated
    GPUs must come out bit for bit the same.  Each side confirms the other."""
    digests = []
    for mode in ("source", "semantic"):
        env = dict(os.environ)
        env.update(MXKV_SIM="1", MXKV_B200_LIBRARY_PATH=sim_lib, MXKV_SIM_DEVICES="4", MXKV_SIM_NORM=mode)
        r = subprocess.run([sys.executable, os.path.join(SIM, "norm_bits_worker.py")], env=env, cwd=ROOT,
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stdout[-1500:] + r.stderr[-1500:]
        digests.append([l for l in r.stdout.splitlines() if l.startswith("DIGEST")][-1])
    assert digests[0] == digests[1]


_ARENA_CASES = [
    (None, "multicast"),
    ("cuMemExportToShareableHandle:1", "ipc"), ("cuMulticastCreate:0", "ipc"), ("cuMulticastBindMem:0", "ipc"),
    ("cuMemMap:1", "ipc"),
    ("cuMemCreate#2:1", "multicast"),            # a LATER segment fails on one rank: that segment is an IPC one everywhere
    ("no_pidfd", "multicast"),                   # pidfd_open refused (EPERM): descriptors travel over unix sockets instead
]
if int(os.environ.get("MXKV_FUZZ_SEEDS", "0")) > 0:      # soak runs: every other stage of the protocol as well
    _ARENA_CASES += [("cuMemCreate:0", "ipc"), ("cuMemImportFromShareableHandle:2", "ipc"), ("cuMulticastAddDevice:1", "ipc"),
                     ("cuMemAddressReserve:2", "ipc"), ("cuMemMap#3:0", "ipc"), ("cuMulticastBindMem:2", "ipc")]


@pytest.mark.parametrize("fail,expect", _ARENA_CASES)
def test_engine_owned_arena_and_its_fallbacks(sim_lib, fail, expect, tmp_path):
    """csrc/vmm_arena.cc on the CPU (tests/sim/fake_driver.cc): three processes build the engine-owned multicast arena
    -- VMM allocations, descriptors handed between the processes with pidfd_getfd or SCM_RIGHTS, one multicast object
    per segment -- and exchange through it; then the same with one driver call failing on one rank at every stage of
    the protocol: every rank must fall back to the cudaMalloc + cudaIpc arena TOGETHER (nobody hangs, nobody keeps a
    half-built segment) and the exchange must still be right."""
    import glob
    world = 3
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="16", WORLD_SIZE=str(world), MXKV_MP_ARENA_ONLY=expect)
    if fail == "no_pidfd":
        shim = os.path.join(os.path.dirname(sim_lib), "libno_pidfd.so")
        env["LD_PRELOAD"] = (env.get("LD_PRELOAD", "") + ":" + shim).strip(":")
        env["MXKV_B200_ARENA_VMM_VERBOSE"] = "1"
    elif fail:
        env["MXKV_SIM_VMM_FAIL"] = fail
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_worker.py")], env=e, cwd=ROOT,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=300)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            for f in glob.glob("/dev/shm/mxkvsim_%d_*" % p.pid):
                os.unlink(f)
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, out[-3000:])
        assert "MP_WORKER_OK rank %d %s" % (r, expect) in out, out[-2000:]


@pytest.mark.parametrize("world", [3, 5, 8])
def test_one_process_per_gpu_under_the_tree_on_simulator(sim_lib, world, tmp_path):
    """MXNET_KVSTORE_USETREE=1 in the torchrun shape (tests/mp_worker.py, tree scenario only): 3, 5 and 8 ranks -- a
    full tree, one with GPUs sitting levels out, the 8-leaf tree -- each running the tree kernel from its own source
    (tests/sim/hostemu_tree.cc) on its shard, with the real flag rendezvous between the ranks."""
    import glob
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world), MXKV_MP_TREE_ONLY="1")
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_worker.py")], env=e, cwd=ROOT,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=900)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            for f in glob.glob("/dev/shm/mxkvsim_%d_*" % p.pid):
                os.unlink(f)
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, out[-3000:])
        assert "MP_WORKER_OK rank %d" % r in out, out[-2000:]


@pytest.mark.parametrize("world,local_world", [(4, 2), (8, 4), (6, 2), (3, 1)])
def test_multi_node_hierarchy_on_simulator(sim_lib, world, local_world, tmp_path):
    """kv.create('dist_device_sync'): `world` processes grouped into nodes of `local_world` (2 x 2, 2 x 4, 3 x 2
    and three single-GPU nodes); inside a node the engine's peer-memory group as above, between the nodes a
    file-based all-reduce where NCCL goes in production.  tests/dist_worker.py checks rank numbering, init from the
    job's rank 0, sums, fused optimizers (bit-exact against the oracle with the hierarchy's association), LAMB,
    and that unsupported combinations are refused."""
    import glob
    env = dict(os.environ)
    env.update(MXKV_SIM="1", MXKV_SIM_MP="1", MXKV_SIM_RDV=str(tmp_path), MXKV_B200_LIBRARY_PATH=sim_lib,
               MXKV_SIM_DEVICES=str(local_world), MXKV_B200_ARENA_MB="256", WORLD_SIZE=str(world),
               MXKV_TEST_LOCAL_WORLD=str(local_world))
    procs = []
    for r in range(world):
        e = dict(env, RANK=str(r), LOCAL_RANK=str(r % local_world))
        procs.append(subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "dist_worker.py")], env=e, cwd=ROOT,
                                      stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    try:
        for p in procs:
            out, _ = p.communicate(timeout=900)
            outs.append(out)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
        for p in procs:
            for f in glob.glob("/dev/shm/mxkvsim_%d_*" % p.pid):
                os.unlink(f)
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d:\n%s" % (r, out[-3000:])
        assert "DIST_WORKER_OK rank %d" % r in out, out[-2000:]
