"""`parallel_run` — the public entry point.

Parity: reference `common/runner.py:139-193` (`parallel_run`: validate
run_option/sync, decide master vs worker from ``PARALLAX_RUN_OPTION``, master
launches and exits, worker returns
``(sess, num_workers, worker_id, num_replicas_per_worker)``) and `:62-137`
(`_parallax_run_master`: mode degeneration, partition-search loop, cleanup).

Differences by design (one process per GPU):
* one worker process per GPU for every run option, so
  ``num_replicas_per_worker`` is always 1 (the reference returns the number of
  local GPUs in PS mode, `ps/runner.py:293-295`);
* a job whose resource spec names a single worker runs in-process (no spawn);
* a process started by ``torchrun`` (RANK/WORLD_SIZE present, no
  PARALLAX_RUN_OPTION) is treated as a worker directly.
"""
import os
import signal
import sys

from . import consts
from . import shard as _shard
from .checkpoint import CheckpointSaver
from .config import ParallaxConfig
from .launcher import launch_workers, kill_all, wait_all
from .log import parallax_log
from .profile import StepProfiler
from .resource import (parse_resource_info, deserialize_resource_info,
                       worker_layout, get_empty_port)
from .session import ParallaxSession


def _as_graph(single_gpu_graph):
    from .graph import Graph
    if isinstance(single_gpu_graph, Graph):
        return single_gpu_graph
    raise TypeError("parallel_run expects a parallax.Graph (model + optimizer "
                    "spec); got %r" % type(single_gpu_graph))


def _run_worker(graph, config, sync, resource_info=None):
    from .parallel.fabric import Comm
    from .parallel.engine import TrainEngine
    comm = Comm.from_env()
    worker_id = int(os.environ.get(consts.PARALLAX_WORKER_ID, comm.rank))
    num_workers = int(os.environ.get(consts.PARALLAX_NUM_WORKERS, comm.world))
    config.set_sync(sync)
    if resource_info is not None:
        config.set_resource_info(resource_info)
    engine = TrainEngine(graph, comm, config, sync=sync)
    _shard.update_shard_values_for_worker(num_workers, worker_id, 1)
    is_chief = worker_id == 0
    saver = None
    if config.ckpt_config.ckpt_dir:
        saver = CheckpointSaver(engine, config.ckpt_config, is_chief)
        saver.restore_if_present()
    profiler = None
    if config.profile_config.profile_dir:
        lrank = int(os.environ.get(consts.PARALLAX_LOCAL_RANK, comm.local_rank))
        profiler = StepProfiler(config.profile_config, worker_id, lrank)
    sess = ParallaxSession(engine, num_workers, worker_id, 1, saver, profiler)
    return sess, num_workers, worker_id, 1


def _parallax_run_master(graph, config, resource_info):
    """Launch the job (and the partition search loop) then return the exit
    code.  Reference `common/runner.py:62-137`."""
    from .analyzer import analyze
    from .partitions import PartitionStatCollector
    run_option = config.normalized_run_option()
    analysis = analyze(graph.model, len(worker_layout(resource_info)))
    run_option = analysis.effective_run_option(run_option)
    num_workers = len(worker_layout(resource_info))
    n_machines = len(resource_info["worker"])

    search = bool(config.search_partitions) and \
        consts.PARALLAX_MIN_PARTITIONS in os.environ and bool(analysis.sparse)
    collector = None
    extra_env = {}
    if search:
        min_p = int(os.environ[consts.PARALLAX_MIN_PARTITIONS])
        port = get_empty_port(1)[0]
        secret = os.urandom(16).hex()
        # workers on other hosts report their step times too: listen on every interface
        # and advertise an address they can reach
        from .resource import all_local, routable_address
        local_job = all_local(resource_info)
        bind = "127.0.0.1:%d" % port if local_job else "0.0.0.0:%d" % port
        addr = "127.0.0.1:%d" % port if local_job else "%s:%d" % (
            routable_address(resource_info["master"][0]["hostname"]), port)
        collector = PartitionStatCollector(max(min_p, n_machines), bind, min_p, authkey=secret)
        collector.setup_manager()
        extra_env[consts.PARALLAX_SEARCH_ADDR] = addr
        extra_env[consts.PARALLAX_SEARCH_AUTHKEY] = secret

    procs = []

    def cleanup(signum=None, frame=None):
        kill_all(procs)

    old = signal.signal(signal.SIGINT, lambda s, f: (cleanup(), sys.exit(130)))
    rc = 0
    try:
        while True:
            if search:
                extra_env[consts.PARALLAX_PARTITIONS] = collector.p_to_test
                extra_env[consts.PARALLAX_SEARCH] = "True"
                parallax_log.info("partition search: trying P=%d",
                                  collector.p_to_test)
            elif collector is not None:
                extra_env[consts.PARALLAX_PARTITIONS] = collector.p_to_test
                extra_env[consts.PARALLAX_SEARCH] = "False"
            del procs[:]
            # fresh rendezvous port per launch
            resource_info["master"][0]["port"] = get_empty_port(1)
            procs.extend(launch_workers(run_option, resource_info, config,
                                        extra_env))
            if not search:
                rc = wait_all(procs)
                break
            search, _ = collector.recv_exec_time(procs, cleanup, num_workers)
    except Exception:
        import traceback
        traceback.print_exc()
        rc = 1
    finally:
        cleanup()
        if collector is not None:
            collector.shutdown()
        signal.signal(signal.SIGINT, old)
    return rc


def parallel_run(single_gpu_graph, resource_info, sync=True,
                 parallax_config=None):
    """Run `single_gpu_graph` data-parallel over the resources in
    `resource_info` (a resource file path or its text).

    Returns ``(session, num_workers, worker_id, num_replicas_per_worker)``.
    In the launcher process this call does not return: it starts the workers
    (which re-execute this script), waits for them and exits.
    """
    config = ParallaxConfig() if parallax_config is None else parallax_config
    run_option = config.normalized_run_option()
    if run_option in ("MPI", "HYBRID") and not sync:
        raise ValueError("run_option %s requires sync=True" % run_option)
    graph = _as_graph(single_gpu_graph)
    config.set_sync(sync)

    role = os.environ.get(consts.PARALLAX_RUN_OPTION)
    if role is not None and role != consts.PARALLAX_RUN_MASTER:
        info = deserialize_resource_info(
            os.environ[consts.PARALLAX_RESOURCE_INFO]) \
            if consts.PARALLAX_RESOURCE_INFO in os.environ else None
        return _run_worker(graph, config, sync, info)

    if role is None and "RANK" in os.environ and "WORLD_SIZE" in os.environ:
        # started by torchrun: already a worker
        return _run_worker(graph, config, sync, None)

    info = parse_resource_info(resource_info, run_option)
    config.set_resource_info(info)
    layout = worker_layout(info)
    if len(layout) == 1:
        gpu = layout[0][3]
        if gpu is not None:
            os.environ.setdefault("LOCAL_RANK", str(gpu))
        return _run_worker(graph, config, sync, info)

    rc = _parallax_run_master(graph, config, info)
    sys.exit(rc)
