"""One-process-per-GPU worker for AdaDelta on the store (tests/test_adadelta.py, simulated runtime): the checks of
tests/adamax_mp_worker.py -- one-shot and two-shot keys, the two sharded states (acc_g, acc_delta) through a checkpoint
on every rank, the multicast kernel, and with MXKV_STEP_OPT_TREE=1 the reference's tree order -- run for AdaDelta."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adamax_mp_worker as W     # noqa: E402
import adadelta_oracle as D      # noqa: E402

KW = dict(learning_rate=1.0, rho=0.95, wd=1e-4, rescale_grad=0.5, clip_gradient=0.7)

if __name__ == "__main__":
    W.main(W.mx.optimizer.AdaDelta, D.OracleAdaDelta, KW, "ADADELTA")
