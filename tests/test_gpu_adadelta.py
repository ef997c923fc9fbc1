"""The AdaDelta optimizer (python/mxnet/optimizer/adadelta.py) fused into the gradient exchange and the native updater:
``AdaDelta.step`` restated in the kernel, against the CPU oracle, bit for bit unless stated, on every dense kernel
variant that serves it.

The tests are tests/test_gpu_adamax.py's, imported here and run with the ``spec`` fixture below; only the options
differ.  AdaDelta's per-key scalars do not depend on the update count, but its states do, so every comparison still
runs over several steps."""
import os
import sys

import pytest

pytestmark = pytest.mark.gpu

import mxnet_b200 as mx

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import adadelta_oracle as D  # noqa: E402
from test_gpu_adamax import Spec  # noqa: E402
from test_gpu_adamax import (  # noqa: E402,F401  (the suite, collected here once more with this file's spec)
    test_forced_variant_whole_sweep_key_set, test_ragged_sizes_and_hyper_parameters_take_effect,
    test_engine_defaults_for_a_c_caller, test_low_precision_keys, test_unaligned_view_takes_the_scalar_path,
    test_cached_launch_plan_replays_with_the_update_count_of_each_step,
    test_deferred_queue_merges_per_key_calls_into_one_launch, test_save_load_round_trip_continues_bit_exact,
    test_get_state_and_set_state, test_native_updater, test_row_sparse_gradient_is_refused,
    test_trainer_modes_match_the_oracle, test_fused_and_python_step_agree,
    test_multi_gpu_one_and_two_shot_keys_with_a_checkpoint, test_tree_sum_feeds_the_update)

ADADELTA = Spec(
    "adadelta", mx.optimizer.AdaDelta, D.OracleAdaDelta,
    kw=dict(learning_rate=1.0, wd=1e-4),
    base=dict(learning_rate=1.0, wd=0.05),
    # rho 0.95 and 0.8: two more double-rounded complements; clip_gradient 0 is on (step clips at 0)
    variants=[dict(rescale_grad=0.14), dict(clip_gradient=0.3), dict(clip_gradient=0.0), dict(learning_rate=0.5),
              dict(rho=0.95), dict(rho=0.8), dict(epsilon=1e-4), dict(wd=0.0)],
    lp_kw=dict(learning_rate=1.0, wd=1e-3, rescale_grad=0.5, clip_gradient=0.6, rho=0.95),
    updater_kw=dict(learning_rate=0.5, wd=1e-2, clip_gradient=0.3, rho=0.95),
    python_kw=dict(learning_rate=1.0, wd=1e-3, clip_gradient=0.01, rho=0.95),
    multi_kw=dict(learning_rate=1.0, wd=1e-4, rescale_grad=0.5, clip_gradient=0.7, rho=0.95))


@pytest.fixture
def spec():
    return ADADELTA
