"""One-process-per-GPU worker for Nadam on the store (tests/test_nadam.py, simulated runtime): the checks of
tests/adamax_mp_worker.py -- one-shot and two-shot keys, the two sharded states (mean, var) through a checkpoint on
every rank, the multicast kernel, and with MXKV_STEP_OPT_TREE=1 the reference's tree order -- run for Nadam.  Every rank
advances the momentum-schedule product over the same keys in the same sorted order, so every rank's weights match the
oracle's bit for bit (within 1e-6 on the multicast kernel); the dumped optimizer carries the product into the store
that loads the checkpoint."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adamax_mp_worker as W     # noqa: E402
import nadam_oracle as N         # noqa: E402

KW = dict(learning_rate=0.002, beta1=0.5, beta2=0.9, schedule_decay=0.008, wd=1e-4, rescale_grad=0.5,
          clip_gradient=0.7)

if __name__ == "__main__":
    W.main(W.mx.optimizer.Nadam, N.OracleNadam, KW, "NADAM")
