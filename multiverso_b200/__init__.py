"""multiverso_b200 -- an H100-native (Hopper, sm_90a) parameter-server engine with the capabilities of
Microsoft/multiverso (tables with Get/Add/GetAsync/AddAsync, server-side updaters, BSP /
async / model-averaging modes, WordEmbedding and LogisticRegression applications)."""
from .api import (aggregate, barrier, dashboard_display, init, is_master_worker, load_table, net_bind,
                  net_connect, net_finalize, num_servers, num_workers, rank, server_id,
                  save_table, server_id_to_rank, set_flag, shutdown, size, symm_tensor, worker_id, worker_id_to_rank,
                  workers_num)
from . import ops, runtime  # noqa: F401
from .tables import (AddOption, ArrayTable, ArrayTableOption, GetOption, HashMatrixTable, KVTable, KVTableOption,
                     MatrixOption, MatrixTable, MatrixTableOption, SparseMatrixTable,
                     SparseMatrixTableOption, create_table)
from .utils import FLAGS, Dashboard, Log

__version__ = "0.1.0"
