"""Sparse-variable partitioning: `get_partitioner` and the online search.

Parity: reference `common/partitions.py:35-51` (`get_partitioner`),
`:53-170` (`PartitionStatCollector`: launch the job with a candidate P, time
steps 50–100, double/halve P, then fit ``t(P) = a·(P-1) + b/P + c`` and pick
the argmin) and `common/session_context.py:28-29,54-71` (workers report the
mean step time of the window to the master).

Fixed relative to the reference (SURVEY §8.4): the `queue` shadowing bug
(`partitions.py:69`) and float partitions from `/` under Python 3
(`:105,112`).

Meaning of P here: a table with P partitions is split row-wise ("mod"
strategy, `embedding_ops.py:151-153`: ``p = id % P, local = id // P``);
partition p is owned by rank ``p % world``.  P therefore controls how rows
interleave across owners and how many independent apply segments each owner
runs; P < world leaves owners idle, large P shrinks per-segment work.
"""
import os
import time
import queue as _queue
from multiprocessing.managers import BaseManager

import numpy as np

from .consts import (PARALLAX_MIN_PARTITIONS, PARALLAX_PARTITIONS,
                     PARALLAX_SEARCH, PARALLAX_SEARCH_AUTHKEY)
from .log import parallax_log


class FixedSizePartitioner(object):
    """The analogue of ``tf.fixed_size_partitioner(P)`` on axis 0."""

    def __init__(self, num_partitions, strategy="mod"):
        assert num_partitions >= 1
        assert strategy in ("mod", "div")
        self.num_partitions = int(num_partitions)
        self.strategy = strategy

    def __call__(self, shape=None, dtype=None):
        return [self.num_partitions] + [1] * (len(shape) - 1 if shape else 0)

    def __repr__(self):
        return "FixedSizePartitioner(%d, %r)" % (self.num_partitions,
                                                 self.strategy)


# every partitioner handed out, so the engine can re-partition in place
# during an in-process search
_issued = []


def get_partitioner(min_num_partitions, strategy="mod"):
    """Return a fixed-size partitioner whose size Parallax decides.

    `min_num_partitions` is the minimum (default) number of partitions that
    fits in memory.  If the launcher is searching, the candidate arrives in
    ``PARALLAX_PARTITIONS``.
    """
    if PARALLAX_MIN_PARTITIONS not in os.environ:
        os.environ[PARALLAX_MIN_PARTITIONS] = str(min_num_partitions)
    if PARALLAX_PARTITIONS in os.environ:
        partitions = int(os.environ[PARALLAX_PARTITIONS])
    else:
        partitions = int(min_num_partitions)
    p = FixedSizePartitioner(partitions, strategy)
    _issued.append(p)
    return p


def issued_partitioners():
    return list(_issued)


def fit_cost_model(p_list, exec_time_list):
    """Least-squares fit of ``t(P) = a·(P-1) + b/P + c``; returns (a, b, c).

    The model is linear in (a, b, c) so a plain lstsq replaces the
    reference's `scipy.optimize.curve_fit` (`partitions.py:155-156`)."""
    P = np.asarray(p_list, dtype=np.float64)
    t = np.asarray(exec_time_list, dtype=np.float64)
    A = np.stack([P - 1.0, 1.0 / P, np.ones_like(P)], axis=1)
    coef, *_ = np.linalg.lstsq(A, t, rcond=None)
    return tuple(float(c) for c in coef)


def find_optimal_p(p_list, exec_time_list):
    """Reference `partitions.py:140-170`."""
    assert len(p_list) == len(exec_time_list) and len(p_list) > 0
    if len(p_list) < 3:
        return int(p_list[int(np.argmin(exec_time_list))])
    max_time = float(max(exec_time_list))
    times = [t / max_time for t in exec_time_list]
    a, b, c = fit_cost_model(p_list, times)
    best_p, best_t = None, None
    for p in range(int(min(p_list)), int(max(p_list)) + 1):
        pred = a * (p - 1) + b / p + c
        if best_t is None or pred < best_t:
            best_p, best_t = p, pred
    return int(best_p)


class SearchState(object):
    """The pure decision logic of the reference's `recv_exec_time`
    (`partitions.py:96-138`), separated from process control so it can be
    unit-tested and reused by the in-process search."""

    def __init__(self, p_to_test, min_partitions=None):
        self.p_to_test = int(p_to_test)
        self.min_partitions = int(min_partitions if min_partitions is not None
                                  else p_to_test)
        self.prev_p = None
        self.prev_exec_time = None
        self.p_list = []
        self.exec_time_list = []
        self.done = False

    def report(self, exec_time, alive=True):
        """Feed the mean step time measured with `p_to_test` (or
        ``alive=False`` if the job died, e.g. OOM).  Returns
        ``(keep_searching, next_p_or_optimal_p)``."""
        stop = False
        if alive:
            curr_p = self.p_to_test
            self.p_list.append(curr_p)
            self.exec_time_list.append(float(exec_time))
            if self.prev_p is not None:
                if self.prev_exec_time < exec_time:
                    if self.prev_p > curr_p:        # got worse while shrinking
                        stop = True
                    else:                           # got worse while growing:
                        self.p_to_test = min(self.p_list) // 2   # try smaller
                else:
                    if self.prev_p < curr_p:
                        self.p_to_test = curr_p * 2
                    else:
                        self.p_to_test = curr_p // 2
                if self.p_to_test < self.min_partitions or \
                        self.p_to_test in self.p_list:
                    stop = True
            else:
                self.p_to_test = curr_p * 2         # increase first
            self.prev_p = curr_p
            self.prev_exec_time = float(exec_time)
        else:
            if self.prev_p is not None:
                stop = True
            else:
                self.p_to_test *= 2
                self.min_partitions = self.p_to_test
        if stop:
            self.done = True
            self.p_to_test = find_optimal_p(self.p_list, self.exec_time_list)
        return (not stop), self.p_to_test


class _QueueManager(BaseManager):
    pass


def _authkey():
    """the job's queue secret: generated by the launcher, handed to the workers through
    the environment"""
    return os.environ.get(PARALLAX_SEARCH_AUTHKEY, "parallax").encode()


class PartitionStatCollector(object):
    """Master-side collector: workers push their window-mean step time to a
    `BaseManager` queue (reference `partitions.py:53-138`)."""

    def __init__(self, p_to_test, address, min_partitions=None, authkey=None):
        self.state = SearchState(p_to_test, min_partitions)
        self.address = address
        self.authkey = (authkey.encode() if isinstance(authkey, str) else authkey) or _authkey()
        self.start = None
        self.m = None
        self._q = None

    @property
    def p_to_test(self):
        return self.state.p_to_test

    def setup_manager(self):
        if self.start is None:
            self.start = time.time()
        q = _queue.Queue()
        self._q = q
        _QueueManager.register("queue", callable=lambda: q)
        host, port = self.address.rsplit(":", 1)
        self.m = _QueueManager(address=("127.0.0.1" if host in ("", "localhost")
                                        else host, int(port)),
                               authkey=self.authkey)
        self.m.start()
        return self.m

    def shutdown(self):
        if self.m is not None:
            try:
                self.m.shutdown()
            except Exception:  # pragma: no cover
                pass
            self.m = None

    def recv_exec_time(self, processes, cleanup, num_required,
                       poll_secs=1.0):
        worker_exec_times = []
        all_alive = True
        q = self.m.queue()
        while len(worker_exec_times) < num_required and all_alive:
            time.sleep(poll_secs)
            while q.qsize() > 0:
                worker_exec_times.append(q.get())
            for p in processes:
                rc = p.poll()
                if rc is not None and rc != 0:
                    all_alive = False
                    break
            if all(p.poll() is not None for p in processes):
                while q.qsize() > 0:
                    worker_exec_times.append(q.get())
                if len(worker_exec_times) < num_required:
                    all_alive = False
        cleanup(None, None)
        ok = all_alive and len(worker_exec_times) > 0
        keep, p = self.state.report(
            float(np.mean(worker_exec_times)) if ok else 0.0, alive=ok)
        if not keep:
            parallax_log.info("optimal partitions: %d, search time: %d secs"
                              % (p, time.time() - self.start))
        return keep, p


def send_exec_time(address, exec_time):
    """Worker side: push this worker's window-mean step time to the master
    (reference `common/session_context.py:64-71`)."""
    host, port = address.rsplit(":", 1)
    _QueueManager.register("queue")
    m = _QueueManager(address=(host, int(port)), authkey=_authkey())
    m.connect()
    m.queue().put(float(exec_time))


def searching():
    return os.environ.get(PARALLAX_SEARCH, "False") == "True"


def search_inprocess(sess, next_feed, min_partitions=None, warmup=5, test=10, sync=None):
    """Online partition search without relaunching the job: for each candidate P
    the engine re-shards its sparse tables in place, runs `warmup + test` training
    steps fed by ``next_feed()`` and times the last `test` (device-synchronised);
    candidates follow the reference's doubling/halving walk and the optimum comes
    from the same cost-model fit (`SearchState`).  Returns the chosen P, with the
    tables left partitioned that way.  Collective: every worker must call it."""
    import time as _time
    import torch
    eng = sess.engine
    if not eng.tables:
        return None
    comm = eng.comm
    cur = max(t.layout.P for t in eng.tables.values())
    p0 = int(min_partitions or os.environ.get(PARALLAX_MIN_PARTITIONS, cur))
    state = SearchState(max(p0, 1), p0)
    keep = True
    while keep:
        p = state.p_to_test
        eng.repartition(p)
        for i in range(warmup + test):
            if i == warmup:
                if comm.is_cuda:
                    torch.cuda.synchronize(comm.device)
                comm.barrier()
                t0 = _time.perf_counter()
            sess.run([eng.graph.loss, "train_op"], next_feed())
        if comm.is_cuda:
            torch.cuda.synchronize(comm.device)
        dt = (_time.perf_counter() - t0) / test
        dts = comm.all_gather_object(dt)
        keep, nxt = state.report(float(np.mean(dts)))
        parallax_log.info("partition search: P=%d  %.3f ms/step", p, 1e3 * float(np.mean(dts)))
    eng.repartition(state.p_to_test)
    parallax_log.info("optimal partitions: %d", state.p_to_test)
    return state.p_to_test
