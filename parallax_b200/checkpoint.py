"""Checkpoint save / restore-on-start.

Parity: reference `common/lib.py:38-56` (`build_ckpt_hooks`: a Saver over all
global variables + `CheckpointSaverHook(save_steps | save_secs)` installed as
a chief-only hook) and the runners passing ``checkpoint_dir`` only on worker 0
so an existing checkpoint is restored automatically at start
(`mpi/runner.py:178-193`, `hybrid/runner.py:243-257`); partitioned variables
are saved as slices of one logical variable (SURVEY §5.4).

Two formats, both layout-independent (resumable under a different world size,
run option or partition count), both named by a ``checkpoint`` index file:

* **sharded** (NVLink fabric, default) — a directory
  ``<ckpt_dir>/model.ckpt-<global_step>/`` with ``manifest.json``, ``dense.pt``
  (chief: full logical dense tensors, slots, EMA, buffers) and one
  ``sparse-<variable>-rank<r>.pt`` per owner holding ``(global row ids, rows,
  slot rows)`` of exactly the rows that rank owns — TF's sharded Saver for
  partitioned variables (`tensorflow/python/training/saver.py:287-433`): no rank
  ever materialises a whole table, so a 100 M-row table saves and restores
  without a gather.  Restore reads its own shard when the placement is unchanged
  and otherwise scatters every shard's rows to their new owners.
* **single file** ``model.ckpt-<global_step>.pt`` (host / library fabric, or
  ``sess_config={"sharded_checkpoint": False}``) — full logical tensors; gathering
  is a collective, only the chief writes.
"""
import json
import re
import os
import time

import torch

from .log import parallax_log

INDEX = "checkpoint"
PREFIX = "model.ckpt-"
MANIFEST = "manifest.json"


def latest_checkpoint(ckpt_dir):
    if not ckpt_dir or not os.path.isdir(ckpt_dir):
        return None
    idx = os.path.join(ckpt_dir, INDEX)
    if os.path.exists(idx):
        with open(idx) as f:
            name = f.read().strip()
        path = os.path.join(ckpt_dir, name)
        if os.path.exists(path):
            return path
    cands = [f for f in os.listdir(ckpt_dir)
             if f.startswith(PREFIX) and (f.endswith(".pt") or os.path.exists(
                 os.path.join(ckpt_dir, f, MANIFEST)))]
    if not cands:
        return None
    cands.sort(key=lambda f: int(re.sub(r"\.pt$", "", f[len(PREFIX):])))
    return os.path.join(ckpt_dir, cands[-1])


def _safe(name):
    return re.sub(r"[^A-Za-z0-9_.-]", "_", name)


def save_sharded(engine, path, is_chief):
    """Write the sharded format into directory `path` (collective)."""
    comm = engine.comm
    if is_chief:
        os.makedirs(path, exist_ok=True)
    comm.barrier()
    if comm.is_cuda:
        torch.cuda.synchronize(comm.device)
    manifest = {"format": 2, "global_step": engine.global_step, "world": comm.world,
                "run_option": engine.run_option, "sparse": {}}
    for name, t in sorted(engine.tables.items()):
        writers = [0] if t.replicated else list(range(comm.world))
        files = ["sparse-%s-rank%d.pt" % (_safe(name), r) for r in writers]
        manifest["sparse"][name] = {
            "V": t.V, "D": t.D, "nslots": t.nslots, "slot_dim": _table_slot_dim(t),
            # rows as the master stores them: "bfloat16" for sparse_weights="bf16" (a
            # manifest without the field holds fp32 rows)
            "weight_dtype": str(getattr(t, "weight_dtype", torch.float32)).replace("torch.", ""),
            "files": files,
            "placement": [t.layout.P, t.layout.strategy, t.layout.world, t.layout.owners,
                          bool(t.replicated)]}
        if comm.rank in writers:
            ids, w = t.local_rows("weight")
            slots = [t.local_rows(str(i))[1] for i in range(t.nslots)]
            fn = os.path.join(path, files[writers.index(comm.rank)])
            torch.save({"ids": ids, "weight": w, "slots": slots}, fn + ".tmp")
            os.replace(fn + ".tmp", fn)
    dense = engine.dense.state_dict() if engine.dense is not None else None   # collective
    if is_chief:
        bufs = {n: b.detach().cpu().clone() for n, b in engine.model.named_buffers()}
        torch.save({"global_step": engine.global_step, "dense": dense, "buffers": bufs},
                   os.path.join(path, "dense.pt"))
        with open(os.path.join(path, MANIFEST + ".tmp"), "w") as f:
            json.dump(manifest, f, indent=1)
        os.replace(os.path.join(path, MANIFEST + ".tmp"), os.path.join(path, MANIFEST))
    comm.barrier()
    return path


def load_sharded(engine, path):
    """Restore from a sharded checkpoint directory (any source world / partitioning)."""
    comm = engine.comm
    with open(os.path.join(path, MANIFEST)) as f:
        manifest = json.load(f)
    d = torch.load(os.path.join(path, "dense.pt"), map_location="cpu", weights_only=False)
    engine.global_step = int(d["global_step"])
    if engine.dense is not None and d.get("dense") is not None:
        engine.dense.load_state_dict(d["dense"])
    bufs = dict(engine.model.named_buffers())
    for n, v in d.get("buffers", {}).items():
        if n in bufs:
            with torch.no_grad():
                bufs[n].copy_(v)
    for name, t in engine.tables.items():
        ent = manifest["sparse"].get(name)
        if ent is None:
            continue
        if ent["V"] != t.V or ent["D"] != t.D:
            raise RuntimeError("checkpoint variable %r has shape (%d, %d), the model (%d, %d)"
                               % (name, ent["V"], ent["D"], t.V, t.D))
        if t.nslots and int(ent["nslots"]) and _slot_dim(ent) != _table_slot_dim(t):
            raise ValueError("checkpoint variable %r has slots of width %d, but its optimizer "
                             "keeps slots of width %d" % (name, _slot_dim(ent),
                                                          _table_slot_dim(t)))
        same = ent["placement"] == [t.layout.P, t.layout.strategy, t.layout.world,
                                    t.layout.owners, bool(t.replicated)]
        files = ent["files"]
        if same and not t.replicated:
            files = [files[comm.rank]]          # my rows are exactly my old shard
        for fn in files:
            sh = torch.load(os.path.join(path, fn), map_location="cpu", weights_only=False)
            if hasattr(t, "load_rows"):
                t.load_rows(sh["ids"], sh["weight"], "weight")
                for i, srows in enumerate(sh["slots"][:t.nslots]):
                    t.load_rows(sh["ids"], srows, str(i))
            else:               # host / library tables: scatter through the logical view
                w, sl = t.full_weight(), t.full_slots()
                w[sh["ids"]] = sh["weight"]
                for i, srows in enumerate(sh["slots"][:len(sl)]):
                    sl[i][sh["ids"]] = srows
                t.load_full(w, sl)
        if hasattr(t, "refresh_shadow"):
            t.refresh_shadow()
    if comm.is_cuda:
        torch.cuda.synchronize(comm.device)
    comm.barrier()
    return manifest


def is_sharded(path):
    return os.path.isdir(path) and os.path.exists(os.path.join(path, MANIFEST))


def list_checkpoints(ckpt_dir):
    """[(global_step, path)] of every checkpoint in `ckpt_dir`, either format, oldest first"""
    out = []
    for f in os.listdir(ckpt_dir):
        if not f.startswith(PREFIX):
            continue
        path = os.path.join(ckpt_dir, f)
        m = re.match(r"^(\d+)(\.pt)?$", f[len(PREFIX):])
        if m and (f.endswith(".pt") or is_sharded(path)):
            out.append((int(m.group(1)), path))
    return sorted(out)


def load_logical(path, max_table_bytes=None):
    """The logical (layout-independent) state dict of a checkpoint in either format — what
    offline consumers (evaluation scripts, checkpoint averaging, the inspection tool) read."""
    if is_sharded(path):
        return assemble_sharded(path, max_table_bytes)
    return torch.load(path, map_location="cpu", weights_only=False)


def read_manifest(path):
    with open(os.path.join(path, MANIFEST)) as f:
        return json.load(f)


def _table_slot_dim(t):
    """Columns of each slot of table `t`: its `slot_dim` (1 for a row-wise optimizer), or D
    for a table that does not declare one."""
    return int(getattr(t, "slot_dim", t.D))


def _slot_dim(ent):
    """Columns of each slot of a manifest entry: D, or 1 for a row-wise optimizer (manifests
    written before row-wise optimizers existed have no "slot_dim": their slots are D wide)."""
    return int(ent.get("slot_dim", ent["D"]))


def assemble_table(path, name, manifest=None):
    """One sparse variable of a sharded checkpoint as full logical tensors
    ``{"weight": [V, D], "slots": [[V, D] or [V, 1] (row-wise), ...]}``, fp32 (bf16 weight
    rows are widened exactly) — no engine, no GPU:
    what an offline tool (`tools/inspect_checkpoint`, an evaluation script on another
    machine) needs."""
    man = manifest or read_manifest(path)
    ent = man["sparse"][name]
    V, D, ns = int(ent["V"]), int(ent["D"]), int(ent["nslots"])
    w, slots, seen = None, None, 0
    for fn in ent["files"]:
        sh = torch.load(os.path.join(path, fn), map_location="cpu", weights_only=False)
        if w is None:
            w = torch.zeros(V, D, dtype=torch.float32)
            slots = [torch.zeros(V, _slot_dim(ent), dtype=s_.dtype) for s_ in sh["slots"][:ns]]
        w[sh["ids"]] = sh["weight"].float()
        for dst, src in zip(slots, sh["slots"]):
            dst[sh["ids"]] = src
        seen += int(sh["ids"].numel())
    if seen != V:
        raise RuntimeError("sharded checkpoint %s: variable %r has %d of %d rows in its shards"
                           % (path, name, seen, V))
    return {"weight": w, "slots": slots}


def assemble_sharded(path, max_table_bytes=None):
    """A sharded checkpoint directory as the single-file logical state dict
    (``global_step`` / ``dense`` / ``buffers`` / ``sparse``).  Tables whose assembled size
    would exceed `max_table_bytes` are left out and listed under ``"skipped"``."""
    man = read_manifest(path)
    d = torch.load(os.path.join(path, "dense.pt"), map_location="cpu", weights_only=False)
    sd = {"global_step": int(d["global_step"]), "dense": d.get("dense"),
          "buffers": d.get("buffers", {}), "sparse": {}, "skipped": []}
    for name, ent in sorted(man["sparse"].items()):
        nbytes = int(ent["V"]) * 4 * (int(ent["D"]) + int(ent["nslots"]) * _slot_dim(ent))
        if max_table_bytes is not None and nbytes > max_table_bytes:
            sd["skipped"].append(name)
            continue
        sd["sparse"][name] = assemble_table(path, name, man)
    return sd


class CheckpointSaver(object):
    """`CheckpointSaverHook` analogue: `after_step` is called by the session
    after every training step on *all* workers."""

    def __init__(self, engine, ckpt_config, is_chief):
        self.engine = engine
        self.dir = ckpt_config.ckpt_dir
        self.save_steps = ckpt_config.save_ckpt_steps
        self.save_secs = ckpt_config.save_ckpt_secs
        self.is_chief = is_chief
        self._last_time = time.time()
        self._last_step = None
        self.enabled = bool(self.dir) and (self.save_steps or self.save_secs)
        self.sharded = (getattr(engine, "backend", None) == "nvlink" and
                        bool(engine.config.sess_option("sharded_checkpoint", True)))

    def restore_if_present(self):
        """Restore-on-start; every rank loads the same logical state and keeps
        its own shard (the reference instead restores on worker 0 and
        broadcasts, `mpi/runner.py:134-139,197`)."""
        if not self.dir:
            return None
        path = latest_checkpoint(self.dir)
        # all ranks must agree on whether a checkpoint exists
        path = self.engine.comm.broadcast_object(path, 0)
        if path is None:
            return None
        if os.path.isdir(path):
            man = load_sharded(self.engine, path)
            step = man["global_step"]
        else:
            sd = torch.load(path, map_location="cpu", weights_only=False)
            self.engine.load_state_dict(sd)
            step = sd["global_step"]
        parallax_log.info("restored checkpoint %s (global_step=%d)", path, step)
        return path

    def _due(self, step):
        if self.save_steps:
            return step % int(self.save_steps) == 0 and step != self._last_step
        if self.save_secs:
            # decision must be identical on all ranks: chief decides
            due = (time.time() - self._last_time) >= float(self.save_secs)
            return bool(self.engine.comm.broadcast_object(due, 0))
        return False

    def after_step(self, step):
        if not self.enabled or not self._due(step):
            return None
        return self.save(step)

    def save(self, step=None):
        step = self.engine.global_step if step is None else step
        if self.sharded:
            name = "%s%d" % (PREFIX, step)
            path = save_sharded(self.engine, os.path.join(self.dir, name), self.is_chief)
            if self.is_chief:
                with open(os.path.join(self.dir, INDEX), "w") as f:
                    f.write(name)
                parallax_log.info("saved sharded checkpoint %s", path)
            self._last_time = time.time()
            self._last_step = step
            return path if self.is_chief else None
        sd = self.engine.state_dict()          # collective
        path = None
        if self.is_chief:
            os.makedirs(self.dir, exist_ok=True)
            name = "%s%d.pt" % (PREFIX, step)
            path = os.path.join(self.dir, name)
            tmp = path + ".tmp"
            torch.save(sd, tmp)
            os.replace(tmp, path)
            with open(os.path.join(self.dir, INDEX), "w") as f:
                f.write(name)
            parallax_log.info("saved checkpoint %s", path)
        self._last_time = time.time()
        self._last_step = step
        return path
