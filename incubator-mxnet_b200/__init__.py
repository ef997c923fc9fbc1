"""H100-native KVStore engine behind MXNet's KVStore API.

Python host side: a ctypes binding of the C ABI in ``include/mxkv_b200.h`` shaped like the
reference's ``python/mxnet/kvstore`` package (``create``, ``KVStoreBase`` registry, native
``KVStore`` wrapper) plus the minimal ``NDArray``/``Context``/``optimizer`` surface that
package needs.  Everything numerical happens in ``libmxkv_b200.so`` (CUDA, sm_90a); there
is no CPU fallback -- calls fail with ``MXNetError`` when no GPU / no native library exists.
"""
from . import base
from .base import MXNetError
from .context import Context, cpu, gpu, cpu_pinned, num_gpus
from . import ndarray
from . import ndarray as nd
from .ndarray import NDArray
from . import optimizer
from . import lr_scheduler
from . import kvstore
from . import kvstore as kv
from .kvstore import KVStore, KVStoreBase, create
from . import dist
from . import topology
from .trainer import Trainer
from . import gluon
from . import context
from . import amp

__version__ = "0.1.0"
