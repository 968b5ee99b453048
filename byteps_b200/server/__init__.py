"""The CPU summation server / scheduler process.

Like the reference (/root/reference/byteps/server/__init__.py:21-27,
launcher/launch.py:234-277) ``import byteps_b200.server`` with
``DMLC_ROLE=server`` or ``scheduler`` runs the role to completion:

    DMLC_ROLE=server DMLC_NUM_WORKER=2 DMLC_NUM_SERVER=1 \
    DMLC_PS_ROOT_URI=127.0.0.1 DMLC_PS_ROOT_PORT=9000 python -c 'import byteps_b200.server'

``DMLC_NUM_WORKER`` counts worker *boxes*; every GPU process of a box is a
transport-level node, so servers/scheduler multiply by ``BYTEPS_LOCAL_SIZE``.
"""
import os


def run(role=None):
    # The engine threads each own an OpenMP team for the summation; idle team members busy-wait by default and
    # then compete with the transport threads for cores (measured on an 8-core host: 74 -> 62 ms per 100 MB
    # push_pull with passive waiting).  libgomp reads this when it is loaded, i.e. before _core is imported.
    os.environ.setdefault("OMP_WAIT_POLICY", "passive")
    from .. import _native

    core = _native.core()
    role = role or os.environ.get("DMLC_ROLE", "server")
    nw = int(os.environ.get("DMLC_NUM_WORKER", "1")) * int(os.environ.get("BYTEPS_LOCAL_SIZE", "1"))
    ns = int(os.environ.get("DMLC_NUM_SERVER", "1"))
    host = os.environ.get("DMLC_PS_ROOT_URI", "127.0.0.1")
    port = int(os.environ.get("DMLC_PS_ROOT_PORT", "9000"))
    node_host = os.environ.get("DMLC_NODE_HOST", "")
    rank = int(os.environ.get("DMLC_SERVER_ID", os.environ.get("DMLC_RANK", "-1")))
    lvl = {"TRACE": 0, "DEBUG": 1, "INFO": 2, "WARNING": 3, "ERROR": 4, "FATAL": 5}.get(
        os.environ.get("BYTEPS_LOG_LEVEL", "WARNING").upper(), 3)
    core.set_log_level(lvl)
    # BYTEPS_SERVER_NUMA_NODE=N: run the whole server (its threads are created below) on NUMA node N and prefer its
    # memory - the socket the GPUs hang off when workers DMA out of the server's store;
    # the same as starting it under `numactl --cpunodebind=N --preferred=N`
    node = os.environ.get("BYTEPS_SERVER_NUMA_NODE", "")
    if role == "server" and node not in ("", "-1"):
        got = core.numa_prefer_node_for_process(int(node))
        core.log(2 if got == 3 else 3, "server: NUMA node %s requested: cpus %s, memory policy %s" % (
            node, "set" if got & 1 else "NOT set", "set" if got & 2 else "NOT set"))
    po = core.Postoffice(role, nw, ns, host, port, node_host, rank if role == "server" else -1, {})
    srv = core.SumServer(po) if role == "server" else None
    recovering = os.environ.get("BYTEPS_RECOVERY", "0") not in ("0", "")
    po.start(0, not recovering)     # a restarted node skips the start barrier
    po.finalize(0, True)            # blocks until every node leaves
    if srv is not None:
        srv.stop()


def byteps_server():
    run("server")


if os.environ.get("DMLC_ROLE", "") in ("server", "scheduler") and os.environ.get("BYTEPS_SERVER_NO_AUTORUN") is None:
    run()
