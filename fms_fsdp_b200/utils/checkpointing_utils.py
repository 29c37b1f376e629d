"""Sharded checkpoint manager with auto-resume.

Capability parity with reference ``fms_fsdp/utils/checkpointing_utils.py:23-316`` and its on-disk
contract (SURVEY.md §5.4):

    <ckpdir>/checkpoints/step_<N>_ckp/
        .metadata, __<rank>_0.distcp ...     torch.distributed.checkpoint (DCP) files, one per writer
        metadata.pth                          {"step": N, "tokens_seen": ..., ...}; marks a sharded ckpt dir
        loader_state_<rank>.pth               one per data-loader worker rank

Tensor keys are the reference's: ``model_state.<fms parameter name>`` and
``optimizer_state.state.<name>.{exp_avg,exp_avg_sq,step}`` + ``optimizer_state.param_groups``, so the
exporters, old checkpoints and third-party DCP tools interoperate, and DCP reshards on load for any
world size.  The engine's *internal* sharding (flat 1-D cuts per unit) is translated at the boundary:
each unit's fp32 shards are all-gathered once and every rank contributes the dim-0 chunk of each
parameter as a ``DTensor(Shard(0))`` -- one unit resident at a time.

Load modes: single ``.pth`` file (weights only, ``strict`` honoured, step/tokens reset) or sharded
directory (model, + optimizer, + loader state); a checkpoint found in the *save* directory wins over
``path`` (job restart => resume step/tokens; otherwise "continued pre-training from someone else's
checkpoint": step 0).
"""
from __future__ import annotations

import os
import shutil
import time
from pathlib import Path
from typing import Any, Dict

import torch
import torch.distributed as dist

from fms_fsdp_b200.parallel.layout import dim0_chunk


def _entries(targdir, qualifier):
    return [os.path.join(targdir, x) for x in os.listdir(targdir) if qualifier(os.path.join(targdir, x))]


def get_latest(targdir, qualifier=lambda x: True, key=os.path.getctime):
    """Full path of the newest qualifying entry of ``targdir`` (None if empty / nonexistent).
    Reference: ``fms_fsdp/utils/checkpointing_utils.py:23-41``."""
    if os.path.exists(targdir) and len(os.listdir(targdir)) > 0:
        cands = _entries(targdir, qualifier)
        if cands:
            return max(cands, key=key)
    return None


def get_oldest(targdir, qualifier=lambda x: True, key=os.path.getctime):
    """Full path of the oldest qualifying entry of ``targdir`` (None if empty / nonexistent).
    Reference: ``fms_fsdp/utils/checkpointing_utils.py:44-62``."""
    if os.path.exists(targdir) and len(os.listdir(targdir)) > 0:
        cands = _entries(targdir, qualifier)
        if cands:
            return min(cands, key=key)
    return None


def resolve_load_path(ckpt_load_path: str) -> str:
    """What ``--ckpt_load_path`` points at.  The reference appends ``checkpoints/`` to a run directory and takes a file as is
    (``main_training_llama.py:121-127``); additionally a single checkpoint folder (``.../step_N_ckp``, holds ``metadata.pth``)
    or a folder of checkpoints is accepted directly instead of silently finding nothing under ``<it>/checkpoints/``."""
    p = ckpt_load_path
    if os.path.isfile(p):
        return p
    if os.path.isdir(p) and not os.path.isdir(os.path.join(p, "checkpoints")):
        names = os.listdir(p)
        if "metadata.pth" in names or any(n.startswith("step_") and n.endswith("_ckp") for n in names):
            return p
    return os.path.join(p, "checkpoints/")


def _step_of(path: str) -> int:
    try:
        return int(os.path.basename(os.path.normpath(path)).split("_")[1])
    except Exception:
        return -1


class Checkpointer:
    """Save / load sharded checkpoints of a ``ShardedModel`` (+ ``ShardedAdamW``, + loader).
    Reference: ``fms_fsdp/utils/checkpointing_utils.py:65-316``."""

    def __init__(self, ckpdir, n_to_save, parallel_mode, rank, local_rank, report_fn=None,
                 model_auto_placement=False):
        self.max_ckps = n_to_save
        self.rank = rank
        self.local_rank = local_rank
        self.ckp_path = os.path.join(ckpdir, "checkpoints/")
        os.makedirs(self.ckp_path, exist_ok=True)
        assert parallel_mode in ["fsdp", "hsdp", "ddp"]
        self.p_mode = parallel_mode
        self.report = self._selective_print if report_fn is None else report_fn
        self.model_auto_placement = model_auto_placement

    # ------------------------------------------------------------------------------------ helpers
    def _selective_print(self, *args, **kwargs):
        if self.rank == 0:
            print(*args)
            for k, v in kwargs.items():
                print(k, "=", v)

    def _cleanup(self):
        """Keep at most ``n_to_save`` ``step_*_ckp`` folders (oldest step removed first)."""
        removed = None
        if self.rank == 0:
            ckps = [x for x in os.listdir(self.ckp_path) if x.startswith("step_") and x.endswith("_ckp")]
            while len(ckps) > self.max_ckps:
                victim = min(ckps, key=lambda x: _step_of(x))
                p = Path(os.path.join(self.ckp_path, victim))
                if p.is_file():
                    p.unlink()
                else:
                    shutil.rmtree(p, ignore_errors=True)
                ckps.remove(victim)
                removed = str(p)
        return removed

    def _validate_ckp_path(self, path):
        """file | sharded dir (has metadata.pth) | dir of checkpoints (newest child) -> path, else None."""
        if path and os.path.exists(path):
            if os.path.isfile(path):
                return path
            names = os.listdir(path)
            if "metadata.pth" in names:
                return path
            if len(names) > 0:
                latest = get_latest(path)
                if os.path.isfile(latest):
                    return latest
                if "metadata.pth" in os.listdir(latest):
                    return latest
        return None

    # ------------------------------------------------------------------- engine <-> DCP translation
    @staticmethod
    def _engine(model):
        return model if hasattr(model, "units") else getattr(model, "_orig_mod", model)

    def _dp_world(self, eng):
        """(writer group, its size, my index in it, am I a writer) for the tensor files."""
        m = eng.mesh
        if m.world == 1:
            return None, 1, 0, True
        if m.shard_size == m.world:
            return dist.group.WORLD, m.world, m.rank, True
        if m.shard_size == 1:  # ddp: fully replicated, rank 0 writes
            return None, 1, 0, m.rank == 0
        # hsdp: the shard group of replica 0 writes (reference: ranks with rank == local_rank, :137-141)
        return m.shard_group, m.shard_size, m.shard_rank, m.replica_rank == 0

    def _wrap(self, full_view: torch.Tensor, group, gsize, gidx):
        """dim-0 chunk of a full parameter as a DTensor(Shard(0)) over the writer group."""
        t = full_view
        if gsize == 1:
            return t.detach().clone().cpu()
        from torch.distributed.device_mesh import DeviceMesh
        from torch.distributed.tensor import DTensor, Shard
        rows = t.shape[0] if t.dim() > 0 else 1
        if t.dim() == 0:
            t = t.reshape(1)
        lo, hi = dim0_chunk(rows, gsize, gidx)
        local = t[lo:hi].detach().clone()
        mesh = self._mesh_for(group, t.device.type)
        return DTensor.from_local(local, mesh, [Shard(0)], run_check=False, shape=t.shape, stride=t.stride())

    def _mesh_for(self, group, device_type):
        from torch.distributed.device_mesh import DeviceMesh
        key = (id(group), device_type)
        cache = self.__dict__.setdefault("_meshes", {})
        if key not in cache:
            cache[key] = DeviceMesh.from_group(group, device_type)
        return cache[key]

    def _collect(self, eng, optimizer, group, gsize, gidx, writer: bool):
        """Build the DCP state dict (collective: every rank participates in the per-unit gathers)."""
        model_state: Dict[str, Any] = {}
        opt_state: Dict[str, Any] = {}
        step = int(getattr(optimizer, "_step", 0)) if optimizer is not None else 0
        for u in eng.units:
            full = eng.gather_unit_full(u, "master")
            for name, v in eng.named_unit_views(u, full):
                if writer:
                    model_state[name] = self._wrap(v, group, gsize, gidx)
            del full
            if optimizer is not None:
                for which in ("exp_avg", "exp_avg_sq"):
                    full = eng.gather_unit_full(u, which)
                    for name, v in eng.named_unit_views(u, full):
                        if writer:
                            opt_state.setdefault(name, {})[which] = self._wrap(v, group, gsize, gidx)
                    del full
                if writer:
                    for s in u.layout.slots:
                        opt_state[s.name]["step"] = torch.tensor(float(step))
        sd: Dict[str, Any] = {"model_state": model_state}
        if optimizer is not None:
            groups = [{k: v for k, v in g.items() if k != "params"} for g in optimizer.param_groups]
            sd["optimizer_state"] = {"state": opt_state, "param_groups": groups}
        return sd

    # --------------------------------------------------------------------------------------- save
    def save(self, step, model, optimizer, dataloader, **kwargs):
        """Sharded DCP checkpoint under ``step_<step>_ckp`` (+ loader state, + ``metadata.pth``)."""
        import torch.distributed.checkpoint as dcp
        from torch.distributed.checkpoint import FileSystemWriter

        eng = self._engine(model)
        save_name = os.path.join(self.ckp_path, "step_" + str(step) + "_ckp")
        t0 = time.time()
        group, gsize, gidx, writer = self._dp_world(eng)
        state_dict = self._collect(eng, optimizer, group, gsize, gidx, writer)
        os.makedirs(save_name, exist_ok=True)
        if writer:
            w = FileSystemWriter(save_name, single_file_per_rank=True)
            if gsize == 1:
                dcp.save(state_dict, storage_writer=w, no_dist=True)
            else:
                dcp.save(state_dict, storage_writer=w, process_group=group)
        del state_dict
        if dataloader is not None:
            dataloader.dataset.save_to_path(save_name)
        if eng.mesh.world > 1:
            dist.barrier()
        if self.rank == 0:
            metadata = dict(kwargs)
            metadata["step"] = step
            torch.save(metadata, os.path.join(save_name, "metadata.pth"))
            # cheap write verification: a silently full disk must not look like a good checkpoint
            ok = os.path.exists(os.path.join(save_name, ".metadata")) and any(
                f.endswith(".distcp") for f in os.listdir(save_name))
            if not ok:
                raise RuntimeError(f"checkpoint {save_name} is incomplete (missing DCP files) -- disk full?")
        self.report(f"Checkpoint saved in {save_name}", model_save_time=time.time() - t0)
        return self._cleanup()

    # --------------------------------------------------------------------------------------- load
    def load(self, model, optimizer, dataloader, path="", reset_stepcount=False, strict=True, is_compiled=False):
        """-> (model, optimizer, dataloader, step, tokens_seen, is_resuming)."""
        import torch.distributed.checkpoint as dcp
        from torch.distributed.checkpoint import FileSystemReader
        from torch.distributed.checkpoint.default_planner import DefaultLoadPlanner

        eng = self._engine(model)
        is_resuming = False
        if self._validate_ckp_path(self.ckp_path) is not None:
            path = self.ckp_path
            is_resuming = True
        load_path = self._validate_ckp_path(path)
        if load_path is None:
            self.report(f"No valid checkpoint detected at {path}, starting from scratch.")
            return model, optimizer, dataloader, 0, 0, False
        self.report(f"Prior checkpoint {load_path} detected.")
        t0 = time.time()

        if os.path.isfile(load_path):
            # memory-mapped: the ranks of a node share the file's page cache instead of each holding a copy
            ckp = torch.load(load_path, map_location="cpu", weights_only=False, mmap=True)
            sd = ckp.get("model_state", ckp)
            sd = sd.get("_orig_mod", sd) if isinstance(sd, dict) and "_orig_mod" in sd else sd
            eng.load_full_state_dict(sd, strict=strict)
            self.report(f"Checkpoint {load_path} is a single-file checkpoint containing only a model. "
                        "Optimizer and dataloader are from scratch.", model_load_time=time.time() - t0)
            return model, optimizer, dataloader, 0, 0, is_resuming

        group, gsize, gidx, _ = self._dp_world(eng)
        if eng.mesh.world > 1 and gsize == 1:
            group, gsize, gidx = None, 1, 0
        reader = FileSystemReader(load_path)
        avail = set(reader.read_metadata().state_dict_metadata.keys())
        prefix = "model_state._orig_mod." if any(k.startswith("model_state._orig_mod.") for k in avail) else "model_state."
        planner = lambda: DefaultLoadPlanner(allow_partial_load=True)  # noqa: E731

        def load_which(which: str, key_of):
            missing = []
            for u in eng.units:
                want, shapes = {}, {}
                for s in u.layout.slots:
                    key = key_of(s.name)
                    if key not in avail:
                        missing.append(key)
                        continue
                    tmpl = torch.zeros(s.shape, dtype=torch.float32, device=eng.device)
                    want[key] = self._wrap(tmpl, group, gsize, gidx) if gsize > 1 else tmpl.cpu()
                    shapes[key] = s
                if not want:
                    continue
                if gsize == 1:
                    dcp.load(want, storage_reader=FileSystemReader(load_path), planner=planner(), no_dist=True)
                    fulls = {shapes[k].name: v.to(eng.device) for k, v in want.items()}
                else:
                    dcp.load(want, storage_reader=FileSystemReader(load_path), planner=planner(), process_group=group)
                    fulls = {shapes[k].name: v.full_tensor() for k, v in want.items()}
                eng.load_unit_from_full(u, which, fulls)
                del want, fulls
            return missing

        missing = load_which("master", lambda n: prefix + n)
        if missing and strict:
            raise RuntimeError(f"checkpoint {load_path} lacks model keys: {missing[:5]} ...")
        self.report(model_load_time=time.time() - t0)

        step, ntok = 0, 0
        if is_resuming:
            metadata = torch.load(os.path.join(load_path, "metadata.pth"), weights_only=False)
            step = metadata.get("step", 0)
            ntok = metadata.get("tokens_seen", 0)
            self.report("Metadata loaded", start_step=step, n_tokens_seen=ntok)

        if optimizer is not None:
            t1 = time.time()
            has_opt = any(k.startswith("optimizer_state.state.") for k in avail)
            if has_opt:
                # checkpoints written under torch.compile carry the wrapper's prefix in the optimizer keys as well
                opfx = "optimizer_state.state._orig_mod." if any(
                    k.startswith("optimizer_state.state._orig_mod.") for k in avail) else "optimizer_state.state."
                for which in ("exp_avg", "exp_avg_sq"):
                    absent = load_which(which, lambda n, w=which: f"{opfx}{n}.{w}")
                    if absent:
                        self.report(f"WARNING: checkpoint has no {which} for {len(absent)} parameters (e.g. {absent[0]}); "
                                    "their moments start from zero")
                step_keys = [k for k in avail if k.startswith("optimizer_state.state.") and k.endswith(".step")]
                if step_keys:
                    holder = {step_keys[0]: torch.zeros(())}
                    dcp.load(holder, storage_reader=FileSystemReader(load_path), planner=planner(),
                             **({"no_dist": True} if eng.mesh.world == 1 else {}))
                    optimizer._step = int(holder[step_keys[0]].item())
                    eng.step_count = optimizer._step
                self.report("Optimizer state loaded", optimizer_load_time=time.time() - t1)
            else:
                self.report("Checkpoint holds no optimizer state; optimizer starts from scratch.")

        if dataloader is not None:
            t2 = time.time()
            dataloader.dataset.load_from_path(load_path)
            self.report("Dataloader state loaded", dataset_load_time=time.time() - t2)
        else:
            self.report("Skipping dataset load, no dataloader provided.")
        if reset_stepcount:
            step = 0
        return model, optimizer, dataloader, step, ntok, is_resuming
