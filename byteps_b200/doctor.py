"""``python -m byteps_b200.doctor``: what this installation can do on this machine.

Prints the build state of the native modules, the GPUs and their peer / multicast capabilities, the transports
that would be selected, and the BytePS / DMLC variables in effect - the first thing to attach to a bug report
(see docs/troubleshooting.md).  Works without a GPU.
"""
from __future__ import annotations

import json
import os
import sys


def collect() -> dict:
    info = {"python": sys.version.split()[0]}
    try:
        import torch

        info["torch"] = torch.__version__
        info["cuda_available"] = bool(torch.cuda.is_available())
        info["torch_cuda"] = torch.version.cuda
        try:
            info["nccl"] = ".".join(str(v) for v in torch.cuda.nccl.version()) if torch.cuda.is_available() else None
        except Exception:  # noqa: BLE001
            info["nccl"] = None
    except Exception as e:  # noqa: BLE001
        info["torch_error"] = repr(e)
        return info
    from . import _native

    try:
        core = _native.core()
        info["core_module"] = getattr(core, "__file__", "?")
        info["compressors"] = sorted(core.compressor_names())
    except Exception as e:  # noqa: BLE001
        info["core_error"] = repr(e)
    try:
        cu = _native.cuda()
        info["cuda_module"] = getattr(cu, "__file__", "?")
        info["max_ranks"] = getattr(cu, "MAX_RANKS", None)
    except Exception as e:  # noqa: BLE001
        info["cuda_module_error"] = repr(e)
    gpus = []
    if info.get("cuda_available"):
        n = torch.cuda.device_count()
        for i in range(n):
            p = torch.cuda.get_device_properties(i)
            peers = [j for j in range(n) if j != i and torch.cuda.can_device_access_peer(i, j)]
            gpus.append({"index": i, "name": p.name, "sm": "%d.%d" % (p.major, p.minor),
                         "memory_gb": round(p.total_memory / 2 ** 30, 1), "sms": p.multi_processor_count,
                         "peer_access": peers})
        info["sm_90_family"] = all(g["sm"] == "9.0" for g in gpus) if gpus else False
    info["gpus"] = gpus
    from .config import Config

    cfg = Config.from_env()
    backend = cfg.backend
    if backend == "auto":
        backend = "local" if cfg.size == 1 else ("symm" if info.get("cuda_available") else "gloo")
        if cfg.is_distributed and cfg.num_server > 0:
            backend = "ps"
    info["selected_backend"] = backend
    info["world"] = {"rank": cfg.rank, "size": cfg.size, "local_rank": cfg.local_rank, "local_size": cfg.local_size,
                     "num_worker": cfg.num_worker, "num_server": cfg.num_server, "distributed": cfg.is_distributed}
    info["nvls_auto"] = bool(info.get("cuda_available")) and cfg.size >= 4 and cfg.use_nvls != "0"
    # CPU-server transport (csrc/net): which van the env selects, and whether the shared-memory van could run here
    van = os.environ.get("DMLC_PS_VAN_TYPE", "tcp") or "tcp"
    if van in ("zmq", "0"):
        van = "tcp"
    if van == "tcp" and os.environ.get("DMLC_LOCAL", "0") not in ("0", ""):
        van = "tcp over Unix-domain sockets (DMLC_LOCAL)"
    try:
        st = os.statvfs("/dev/shm")
        shm_free_mb = st.f_bavail * st.f_frsize >> 20
        stale = len([f for f in os.listdir("/dev/shm") if f.startswith("bps_shmvan_")])
    except OSError:
        shm_free_mb, stale = None, 0
    info["transport"] = {"van": van, "lanes": int(os.environ.get("DMLC_NUM_PORTS", "2") or 2),
                         "ipc": os.environ.get("BYTEPS_ENABLE_IPC", "0") not in ("0", "") or van == "shm",
                         "dev_shm_free_mb": shm_free_mb, "shmvan_objects": stale,
                         "c_api_library": os.path.exists(os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                                                      "libbyteps_b200.so"))}
    info["env"] = {k: v for k, v in sorted(os.environ.items())
                   if k.startswith(("BYTEPS_", "DMLC_", "PS_")) or k in ("RANK", "WORLD_SIZE", "LOCAL_RANK",
                                                                        "MASTER_ADDR", "MASTER_PORT",
                                                                        "NVIDIA_VISIBLE_DEVICES", "CUDA_VISIBLE_DEVICES")}
    return info


def main(argv=None) -> int:
    argv = list(sys.argv[1:] if argv is None else argv)
    if "--reap-shm" in argv:
        # unlink /dev/shm/BytePS_* objects whose creating pid is gone (csrc/net/van.cc: ShmRegistry::reap_stale)
        from . import _native

        n = _native.core().shm_reap_stale("/dev/shm")
        print("removed %d shared-memory object(s) of dead byteps processes" % n)
        return 0
    info = collect()
    if "--json" in argv:
        print(json.dumps(info, indent=1, default=str))
        return 0
    print("byteps_b200 doctor")
    print("  python %s, torch %s (CUDA %s), NCCL %s" % (info.get("python"), info.get("torch"), info.get("torch_cuda"),
                                                     info.get("nccl")))
    print("  native runtime : %s" % info.get("core_module", info.get("core_error")))
    print("  CUDA module    : %s" % info.get("cuda_module", info.get("cuda_module_error")))
    if not info.get("gpus"):
        print("  GPUs           : none visible -> gloo / CPU-server transports only")
    for g in info.get("gpus", []):
        print("  GPU %d          : %s, sm_%s, %.0f GB, %d SMs, peer access to %s" % (
            g["index"], g["name"], g["sm"].replace(".", ""), g["memory_gb"], g["sms"], g["peer_access"] or "nobody"))
    if info.get("gpus") and not info.get("sm_90_family"):
        print("  WARNING        : the kernels are built for sm_90a only; they will not load on these GPUs")
    w = info["world"]
    print("  topology       : rank %d of %d (local %d of %d), %d worker box(es), %d server(s)%s" % (
        w["rank"], w["size"], w["local_rank"], w["local_size"], w["num_worker"], w["num_server"],
        ", CPU-server mode" if w["distributed"] else ""))
    print("  backend        : %s%s" % (info["selected_backend"], " (NVLS multicast attempted)" if info["nvls_auto"] else ""))
    t = info["transport"]
    print("  PS transport   : van=%s, %d lane(s), colocated IPC %s; /dev/shm %s MB free, %d shm-van object(s) present; "
          "C API library %s" % (t["van"], t["lanes"], "on" if t["ipc"] else "off", t["dev_shm_free_mb"],
                                t["shmvan_objects"], "built" if t["c_api_library"] else "missing"))
    if info["env"]:
        print("  environment    :")
        for k, v in info["env"].items():
            print("      %s=%s" % (k, v))
    return 0


if __name__ == "__main__":
    sys.exit(main())
