"""Environment-variable configuration.

The reference reads ~95 environment variables ad hoc (SURVEY 5.6,
/root/reference/docs/env.md).  The ones that still make sense on a single
NVSwitch box keep their names; torchrun's RANK/WORLD_SIZE/LOCAL_RANK are
accepted as an alternative bootstrap.  New knobs are prefixed BYTEPS_ too.
"""
import os
from dataclasses import dataclass, field


def _i(name, default):
    v = os.environ.get(name)
    return int(v) if v not in (None, "") else default


def _f(name, default):
    v = os.environ.get(name)
    return float(v) if v not in (None, "") else default


def _b(name, default=False):
    v = os.environ.get(name)
    if v in (None, ""):
        return default
    return v.lower() not in ("0", "false", "no", "off")


def _s(name, default=""):
    v = os.environ.get(name)
    return v if v not in (None, "") else default


@dataclass
class Config:
    # ---- topology / bootstrap
    role: str = "worker"
    rank: int = 0
    size: int = 1
    local_rank: int = 0
    local_size: int = 1
    worker_id: int = 0
    num_worker: int = 1
    num_server: int = 0
    root_uri: str = "127.0.0.1"
    root_port: int = 9000
    # ---- performance
    partition_bytes: int = 4096000
    group_bytes: int = 32 << 20          # bytes fused into one kernel launch
    scheduling_credit: int = 0           # 0 = unlimited (reference default: scheduling off)
    min_compress_bytes: int = 65536
    key_hash_fn: str = "djb2"
    enable_async: bool = False
    force_distributed: bool = False
    omp_threads: int = 4
    threadpool_size: int = 4
    server_engine_threads: int = 4
    # ---- H100 data path
    backend: str = "auto"                # auto | symm | nccl | gloo | ps | local
    symm_mode: str = "auto"              # auto | vmm | ipc
    arena_bytes: int = 256 << 20
    use_nvls: str = "auto"               # auto | 0 | 1
    one_shot_bytes: int = 256 << 10      # <= this -> one-shot kernel
    comm_blocks: int = 0                 # 0 = heuristic
    comm_threads: int = 512
    wire_dtype: str = ""                 # "", "bf16", "fp16": cast on the wire
    # ---- debug / trace
    log_level: str = "WARNING"
    trace_on: bool = False
    trace_start_step: int = 10
    trace_end_step: int = 20
    trace_dir: str = "./trace"
    telemetry_on: bool = True
    debug_sample_tensor: str = ""
    extras: dict = field(default_factory=dict)

    @staticmethod
    def from_env() -> "Config":
        c = Config()
        e = os.environ
        c.role = _s("DMLC_ROLE", "worker")
        # torchrun-style first, BytePS/DMLC-style second
        if "RANK" in e and "WORLD_SIZE" in e and "BYTEPS_LOCAL_RANK" not in e:
            c.rank = _i("RANK", 0)
            c.size = _i("WORLD_SIZE", 1)
            c.local_rank = _i("LOCAL_RANK", c.rank)
            c.local_size = _i("LOCAL_WORLD_SIZE", c.size)
            c.worker_id = _i("GROUP_RANK", c.rank // max(c.local_size, 1))
            c.num_worker = max(1, c.size // max(c.local_size, 1))
        else:
            c.local_rank = _i("BYTEPS_LOCAL_RANK", 0)
            c.local_size = _i("BYTEPS_LOCAL_SIZE", 1)
            c.worker_id = _i("DMLC_WORKER_ID", 0)
            c.num_worker = _i("DMLC_NUM_WORKER", 1)
            c.rank = _i("BYTEPS_GLOBAL_RANK", c.local_rank + c.worker_id * c.local_size)
            c.size = c.num_worker * c.local_size
        c.num_server = _i("DMLC_NUM_SERVER", 0)
        c.root_uri = _s("DMLC_PS_ROOT_URI", _s("MASTER_ADDR", "127.0.0.1"))
        c.root_port = _i("DMLC_PS_ROOT_PORT", 9000)
        c.partition_bytes = _i("BYTEPS_PARTITION_BYTES", 4096000)
        c.group_bytes = _i("BYTEPS_GROUP_BYTES", 32 << 20)
        c.scheduling_credit = _i("BYTEPS_SCHEDULING_CREDIT", 0)
        c.min_compress_bytes = _i("BYTEPS_MIN_COMPRESS_BYTES", 65536)
        c.key_hash_fn = _s("BYTEPS_KEY_HASH_FN", "djb2")
        c.enable_async = _b("BYTEPS_ENABLE_ASYNC")
        c.force_distributed = _b("BYTEPS_FORCE_DISTRIBUTED")
        c.omp_threads = _i("BYTEPS_OMP_THREAD_PER_GPU", 4)
        c.threadpool_size = _i("BYTEPS_THREADPOOL_SIZE", 4)
        c.server_engine_threads = _i("BYTEPS_SERVER_ENGINE_THREAD", 4)
        c.backend = _s("BYTEPS_BACKEND", "auto")
        c.symm_mode = _s("BYTEPS_SYMM_BACKEND", "auto")
        c.arena_bytes = _i("BYTEPS_ARENA_BYTES", 256 << 20)
        c.use_nvls = _s("BYTEPS_USE_NVLS", "auto")
        c.one_shot_bytes = _i("BYTEPS_ONE_SHOT_BYTES", 256 << 10)
        c.comm_blocks = _i("BYTEPS_COMM_BLOCKS", 0)
        c.comm_threads = _i("BYTEPS_COMM_THREADS", 512)
        c.wire_dtype = _s("BYTEPS_WIRE_DTYPE", "")
        c.log_level = _s("BYTEPS_LOG_LEVEL", "WARNING")
        c.trace_on = _b("BYTEPS_TRACE_ON")
        c.trace_start_step = _i("BYTEPS_TRACE_START_STEP", 10)
        c.trace_end_step = _i("BYTEPS_TRACE_END_STEP", 20)
        c.trace_dir = _s("BYTEPS_TRACE_DIR", "./trace")
        c.telemetry_on = _b("BYTEPS_TELEMETRY_ON", True)
        c.debug_sample_tensor = _s("BYTEPS_DEBUG_SAMPLE_TENSOR", "")
        return c

    @property
    def is_distributed(self) -> bool:
        """CPU-server mode: the reference's `_is_distributed_job`
        (/root/reference/byteps/common/global.cc:149-152)."""
        return self.num_worker > 1 and self.num_server > 0 or self.force_distributed

    def partition_bound(self, page: int = 4096) -> int:
        """Partition byte bound rounded up to local_size*page so shards stay
        page/vector aligned (global.cc:142)."""
        m = max(1, self.local_size) * page
        return ((self.partition_bytes + m - 1) // m) * m
