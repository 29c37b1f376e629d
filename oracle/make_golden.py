"""Record what the original fms-fsdp project computes, as the golden data the comparison tests check against.

    python oracle/make_golden.py --reference /path/to/fms-fsdp-checkout

Writes ``tests/golden/reference_*.json.gz`` (and the reference-written loader checkpoints under
``tests/golden/reference_ckpt/``).  The tests never import the original project: they compare this repository's output
with these recordings.  Re-run only when a recording has to change on purpose (e.g. a new comparison case).
"""
from __future__ import annotations

import argparse
import ast
import dataclasses
import gzip
import importlib.util
import json
import os
import shutil
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _dump(name, obj):
    """gzip without a timestamp, so re-recording unchanged content leaves the files byte-identical."""
    os.makedirs(GOLDEN, exist_ok=True)
    data = json.dumps(obj, sort_keys=True, separators=(",", ":")).encode()
    with open(os.path.join(GOLDEN, name), "wb") as raw, gzip.GzipFile(fileobj=raw, mode="wb", mtime=0, filename="") as f:
        f.write(data)


def record_api(ref):
    """Public names and parameter lists of the modules whose API this repository mirrors."""
    import test_api_parity as T
    out = {}
    for path in sorted(T.MODULES):
        tree = ast.parse(open(os.path.join(ref, path)).read())
        fns, classes = {}, {}
        names = []
        for node in tree.body:
            if isinstance(node, ast.FunctionDef) and not node.name.startswith("_"):
                names.append(node.name)
                fns[node.name] = list(T._positional_names(node))
            elif isinstance(node, ast.ClassDef):
                meth = {b.name: list(T._positional_names(b)) for b in node.body if isinstance(b, ast.FunctionDef)
                        and (b.name == "__init__" or not b.name.startswith("_"))}
                classes[node.name] = meth
                if not node.name.startswith("_"):
                    names.append(node.name)
            elif isinstance(node, ast.Assign):
                names += [t.id for t in node.targets if isinstance(t, ast.Name) and not t.id.startswith("_")]
        out[path] = {"names": names, "functions": fns, "classes": classes}
    _dump("reference_api.json.gz", out)


def record_sources(ref):
    """SHA-256 of every ``fms_fsdp/**/*.py`` file of the original project (what the benchmark's reference arm must run)."""
    import hashlib
    out = {}
    for dirpath, _, files in os.walk(os.path.join(ref, "fms_fsdp")):
        for f in files:
            if f.endswith(".py"):
                path = os.path.join(dirpath, f)
                out[os.path.relpath(path, ref)] = hashlib.sha256(open(path, "rb").read()).hexdigest()
    _dump("reference_sources.json.gz", out)


def record_config(ref):
    """Model zoo, train_config defaults and the synthetic loader stream of the original project."""
    import re
    src = os.path.join(ref, "fms_fsdp", "utils", "config_utils.py")
    variants = sorted(set(re.findall(r'model_variant == "([a-z0-9_.]+)"', open(src).read())))
    code = (
        "import sys, json, dataclasses\n"
        f"sys.path = [{ref!r}, {os.path.join(ROOT, 'baseline', 'fms_shim')!r}] + [p for p in sys.path if p not in ('', {ROOT!r})]\n"
        "from fms_fsdp.utils.config_utils import get_model_config\n"
        "from fms_fsdp.config import train_config\n"
        "from fms_fsdp.utils.dataloader_utils import get_dummy_loader\n"
        "zoo = {}\n"
        f"for v in {variants!r}:\n"
        "    c = get_model_config(v)\n"
        "    zoo[v] = c if isinstance(c, dict) else dataclasses.asdict(c)\n"
        "c = train_config(); c.seq_length, c.batch_size, c.vocab_size = 16, 2, 50\n"
        "it = iter(get_dummy_loader(c, 1, 4))\n"
        "batches = [[t.tolist() for t in next(it)] for _ in range(5)]\n"
        "print('OUT' + json.dumps({'zoo': zoo, 'cfg': dataclasses.asdict(train_config()), 'batches': batches}))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd="/", timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    _dump("reference_config.json.gz", json.loads(r.stdout.split("OUT", 1)[1]))


def record_selective_ac(ref):
    """Which blocks the original ``apply_fsdp_checkpointing`` wraps, for the depths / fractions of
    tests/test_selective_ac.py."""
    import test_selective_ac as T
    code = (
        "import sys, json\n"
        f"sys.path = [{ref!r}] + [p for p in sys.path if p not in ('', {ROOT!r})]\n"
        "import importlib.util, torch.nn as nn\n"
        f"spec = importlib.util.spec_from_file_location('ref_ac', {os.path.join(ref, 'fms_fsdp', 'policies', 'ac_handler.py')!r})\n"
        "ac = importlib.util.module_from_spec(spec); spec.loader.exec_module(ac)\n"
        "from torch.distributed.algorithms._checkpoint.checkpoint_wrapper import CheckpointWrapper\n"
        "class Blk(nn.Linear):\n    pass\n"
        "out = {}\n"
        f"for n in {T.AC_DEPTHS!r}:\n"
        f"    for p in {T.AC_FRACTIONS!r}:\n"
        "        m = nn.Sequential(*[Blk(2, 2) for _ in range(n)])\n"
        "        ac.apply_fsdp_checkpointing(m, Blk, p)\n"
        "        out[f'{n}:{p}'] = [isinstance(c, CheckpointWrapper) for c in m]\n"
        "print('OUT' + json.dumps(out))\n")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd="/", timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    _dump("reference_selective_ac.json.gz", json.loads(r.stdout.split("OUT", 1)[1]))


def record_datasets(ref):
    """Token streams and loader checkpoints of the original dataset classes on the corpora of tests/test_datasets.py."""
    import torch

    import fms_fsdp_b200.utils.dataset_utils as OURS
    import test_datasets as T
    spec = importlib.util.spec_from_file_location("_reference_dataset_utils",
                                                  os.path.join(ref, "fms_fsdp", "utils", "dataset_utils.py"))
    REF = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(REF)
    corpus = T.corpus.__wrapped__()
    lines = lambda it, n: [list(map(int, next(it))) for _ in range(n)]   # noqa: E731
    out = {}
    ck_root = os.path.join(GOLDEN, "reference_ckpt")
    shutil.rmtree(ck_root, ignore_errors=True)

    # full stack: stream, continuation of OUR world-2 checkpoint at world 2, and the reference's own world-2 checkpoint
    out["full_stack"] = lines(iter(T._full_stack(REF, corpus, 0, 1)), 300)
    tmp = tempfile.mkdtemp()
    stacks = [T._full_stack(OURS, corpus, r, 2) for r in range(2)]
    for s in stacks:
        T.take(iter(s), 40)
    for s in stacks:
        s.save_to_path(os.path.join(tmp, "ours"))
    resumed = [T._full_stack(REF, corpus, r, 2) for r in range(2)]
    for s in resumed:
        s.load_from_path(os.path.join(tmp, "ours"))
    out["ours_to_ref"] = [lines(iter(s), 60) for s in resumed]
    stacks = [T._full_stack(REF, corpus, r, 2) for r in range(2)]
    for s in stacks:
        T.take(iter(s), 40)
    for s in stacks:
        s.save_to_path(os.path.join(ck_root, "full_stack_w2"))
    resumed = [T._full_stack(REF, corpus, r, 4) for r in range(4)]
    for s in resumed:
        s.load_from_path(os.path.join(ck_root, "full_stack_w2"))
    out["ref_w2_to_w4"] = [lines(iter(s), 60) for s in resumed]

    # parquet + arrow reader
    tmpt, docs, vocab = T.text_corpus.__wrapped__()
    theirs = REF.StreamingDocDataset(f"{tmpt}/data/mix", 0, 1, REF.AutoHandler(f"{tmpt}/tok", "text"), 0, strip_tokens={1, 2},
                                     seed=3, max_chunksize=16)
    out["auto_reader"] = lines(iter(theirs), 200)

    # line packer modes
    out["line_packer"] = []
    for kw in T.PACKER_MODES:
        d = REF.StreamingDocDataset(corpus, 0, 1, REF.ArrowHandler(), -1, seed=11, max_chunksize=40)
        d = REF.SamplingDataset(corpus, d, -1, datasets=["dataset_1", "dataset_2"], weights=[1, 2], verbose=False)
        out["line_packer"].append(lines(iter(REF.BufferDataset(d, 37, **kw)), 250))

    # reader partitioning
    out["partitioning"] = {}
    for world, rank, bos, min_len, nlog in T.PARTITION_CASES:
        if min_len >= 60:
            continue
        d = REF.StreamingDocDataset(os.path.join(corpus, "dataset_2"), rank, world, REF.ArrowHandler(), -1, bos_token=bos,
                                    min_length=min_len, seed=5, max_chunksize=33)
        out["partitioning"][f"{world},{rank},{bos},{min_len},{nlog}"] = lines(
            iter(REF.ScalableShardDataset(d, -1, n_logical_shards=nlog * world)), 150)

    # rescaled resume: continuation of the reference at new_world from a checkpoint written at old_world
    out["rescaled"] = {}
    for writer_is_ours, old_world, new_world in T.RESCALE_CASES:
        writer = OURS if writer_is_ours else REF
        key = f"{int(writer_is_ours)},{old_world},{new_world}"
        ck = os.path.join(ck_root, f"rescale_{old_world}") if not writer_is_ours else os.path.join(tmp, key)
        olds = [T._rescale_stack(writer, corpus, r, old_world) for r in range(old_world)]
        for s in olds:
            T.take(iter(s), 30)
        for s in olds:
            s.save_to_path(ck)
        res = []
        for r in range(new_world):
            b = T._rescale_stack(REF, corpus, r, new_world)
            b.load_from_path(ck)
            res.append(lines(iter(b), 40))
        out["rescaled"][key] = res

    # multi-worker DataLoader: batches and the names of the auto-checkpoints
    ldr = T._worker_loader(REF, corpus, os.path.join(tmp, "ref"))
    it = iter(ldr)
    out["multi_worker"] = [next(it).tolist() for _ in range(24)]
    del it
    ckd = os.path.join(tmp, "ref", "checkpoints")
    steps = sorted(os.listdir(ckd))
    out["multi_worker_ckpts"] = {"steps": steps, "last": sorted(os.listdir(os.path.join(ckd, steps[-1])))}
    _dump("reference_datasets.json.gz", out)
    del torch


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", required=True, help="checkout of the original fms-fsdp project")
    a = ap.parse_args()
    record_api(a.reference)
    record_sources(a.reference)
    record_config(a.reference)
    record_selective_ac(a.reference)
    record_datasets(a.reference)
    print("golden data written under", GOLDEN)
