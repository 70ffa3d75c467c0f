"""Autotuner (Python face of `ops/csrc/runtime/autotune.cpp`).

``PARALLAX_AUTOTUNE=1`` makes the engine tune its communication knobs during
the first steps (Horovod: ``HOROVOD_AUTOTUNE``, CSV log via
``HOROVOD_AUTOTUNE_LOG`` — `horovod/common/parameter_manager.cc:96-101`).
Knobs must be identical on all ranks (the per-CTA barrier slots depend on the
grid size), so rank 0 decides and the values are broadcast through the
control plane each time they change.
"""
import ctypes
import os
import time

from .. import ops
from ..consts import PARALLAX_AUTOTUNE, PARALLAX_AUTOTUNE_LOG

_i, _d = ctypes.c_int, ctypes.c_double
_pd, _pi = ctypes.POINTER(ctypes.c_double), ctypes.POINTER(ctypes.c_int)
ops.register_signatures({
    "px_autotune_create": (_i, [_i, _pd, _pd, _i, _pi, _i, _i, _i, ctypes.c_uint]),
    "px_autotune_current": (_i, [_i, _pd, _pi]),
    "px_autotune_report": (_i, [_i, _d]),
    "px_autotune_num_points": (_i, [_i]),
    "px_autotune_best_score": (_d, [_i]),
    "px_autotune_destroy": (_i, [_i]),
})


class BayesianTuner(object):
    """Continuous knobs ``{name: (lo, hi)}`` searched jointly by GP/EI, then
    categorical knobs ``{name: [values]}`` swept one after the other."""

    def __init__(self, continuous, categorical=None, samples_per_point=5,
                 max_points=20, warmups=3, seed=1):
        self.L = ops.lib()
        self.cnames = list(continuous)
        self.knames = list(categorical or {})
        self.kvalues = [list(categorical[k]) for k in self.knames]
        nd, nk = len(self.cnames), len(self.knames)
        lo = (ctypes.c_double * max(nd, 1))(*[continuous[n][0] for n in self.cnames])
        hi = (ctypes.c_double * max(nd, 1))(*[continuous[n][1] for n in self.cnames])
        ks = (ctypes.c_int * max(nk, 1))(*[len(v) for v in self.kvalues])
        self.h = self.L.px_autotune_create(nd, lo, hi, nk, ks, samples_per_point,
                                           max_points, warmups, seed)
        self._x = (ctypes.c_double * max(nd, 1))()
        self._k = (ctypes.c_int * max(nk, 1))()
        self.done = False

    def current(self):
        rc = self.L.px_autotune_current(self.h, self._x, self._k)
        self.done = rc == 1
        out = {n: self._x[i] for i, n in enumerate(self.cnames)}
        out.update({n: self.kvalues[i][self._k[i]] for i, n in enumerate(self.knames)})
        return out

    def report(self, score):
        rc = self.L.px_autotune_report(self.h, float(score))
        if rc == 2:
            self.done = True
        return rc

    def num_points(self):
        return self.L.px_autotune_num_points(self.h)

    def best_score(self):
        return self.L.px_autotune_best_score(self.h)

    def close(self):
        self.L.px_autotune_destroy(self.h)


class EngineAutotuner(object):
    """Tunes the engine's communication knobs in the regime production runs in.

    Horovod's parameter manager scores a setting by bytes/µs over a few cycles of the
    running job (`horovod/common/parameter_manager.cc:155-181`) and tunes the fusion
    threshold x cycle time jointly plus categorical switches (`:45-56`).  Here every
    candidate setting is applied, the training step is RE-CAPTURED into a CUDA graph
    (after the usual eager warm-up steps) and scored by the device time of `MEASURE`
    graph replays — so the numbers the tuner sees are the numbers the job will run at.
    Knobs: CTAs of the dense comm kernels, CTA cap of the sparse kernels (continuous,
    GP/EI), then the schedule switches one by one (categorical): sparse push from inside
    backward vs after it, last dense bucket held back behind the sparse push or not.  Every
    knob is an attribute of the engine, its fabric or its groups.  Rank 0 decides; values
    are broadcast so every rank applies the same setting at the same step."""
    MEASURE = 8

    def __init__(self, engine):
        self.engine = engine
        self.tuner = BayesianTuner(
            {"comm_blocks": (4.0, 128.0), "sparse_blocks": (16.0, 296.0)},
            categorical={"early_push": [True, False], "defer_last": [True, False]},
            samples_per_point=1, warmups=0, max_points=10) if engine.comm.rank == 0 else None
        self.log = os.environ.get(PARALLAX_AUTOTUNE_LOG)
        self.done = False
        self.best = None
        self._since = 0
        self._ev = None
        self._apply(self._decide())

    @staticmethod
    def wanted():
        return os.environ.get(PARALLAX_AUTOTUNE, "0") not in ("0", "", "false", "False")

    def _decide(self):
        vals = None
        if self.tuner is not None:
            cur = self.tuner.current()
            vals = dict(cur, comm_blocks=int(round(cur["comm_blocks"])),
                        sparse_blocks=int(round(cur["sparse_blocks"])), done=self.tuner.done)
        return self.engine.comm.broadcast_object(vals, 0)

    def _apply(self, vals):
        eng = self.engine
        eng.fabric.max_blocks = max(1, min(128, vals["comm_blocks"]))
        eng.fabric.dense_blocks = max(1, 4 * vals["comm_blocks"])      # 16 .. 512 CTAs
        for grp in getattr(eng, "sparse_groups", ()):
            grp.max_blocks = max(1, vals["sparse_blocks"])
            grp.early_push = bool(vals["early_push"])
        if eng.dense is not None:
            eng.dense.defer_last = bool(vals["defer_last"])
        self.current = {k: v for k, v in vals.items() if k != "done"}
        self.done = bool(vals["done"])
        # the captured graph (if any) bakes the old grids / schedule in: capture again
        eng._graph_state = None
        self._warm = int(eng.config.sess_option("graph_warmup", 3)) if eng._use_graph_possible() \
            else 1
        eng._graph_not_before = eng.global_step + self._warm
        self._since = 0
        if self.log and eng.comm.rank == 0:
            with open(self.log, "a") as f:
                f.write("%d,%s\n" % (eng.global_step, ",".join(
                    "%s=%s" % kv for kv in sorted(vals.items()))))

    def step_begin(self):
        import torch
        # steps 0..warm-1: eager warm-up; step warm: capture (+ first replay); then MEASURE
        # replays timed on the device
        if not self.done and self._since == self._warm + 1:
            self._ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self._ev[0].record()

    def step_end(self):
        if self.done:
            return
        self._since += 1
        if self._since < self._warm + 1 + self.MEASURE:
            return
        self._ev[1].record()
        self._ev[1].synchronize()
        ms = self._ev[0].elapsed_time(self._ev[1]) / self.MEASURE
        import torch
        t = torch.tensor([ms], device=self.engine.comm.device)
        if self.engine.comm.distributed:
            import torch.distributed as dist
            dist.all_reduce(t, op=dist.ReduceOp.MAX, group=self.engine.comm.group)
        ms = float(t.item())
        if self.best is None or ms < self.best[0]:
            self.best = (ms, dict(self.current))
        if self.tuner is not None:
            self.tuner.report(1.0 / max(ms, 1e-6))
        vals = self._decide()
        if vals["done"] and self.best is not None:
            vals = dict(self.best[1], done=True)      # settle on the best setting seen
            vals = self.engine.comm.broadcast_object(vals, 0)
        self._apply(vals)
