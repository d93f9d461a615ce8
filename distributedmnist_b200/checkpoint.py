"""Checkpoint writer/reader with the reference's directory contract.

reference: ``tf.train.Saver()`` over all global variables (8 model tensors +
``global_step``) driven by the Supervisor every ``save_interval_secs`` plus one
final explicit save (src/distributed_train.py:222,244-252,405-408); the
evaluator resolves the ``checkpoint`` state file, accepts absolute or relative
``model_checkpoint_path`` and derives the step from the suffix after the last
``-`` (src/nn_eval.py:70-88).

Kept compatible: ``train_dir/checkpoint`` text-proto state file,
``model.ckpt-<global_step>`` prefix, TF's three-file naming
(``.index`` / ``.data-00000-of-00001``), the variable-name map
(``global_step``, ``Variable`` .. ``Variable_7``), TF variable layouts, and
``max_to_keep=5`` retention.  The payload container is our own (a JSON index +
raw little-endian tensor bytes): no TensorFlow exists here to read a TF bundle,
so byte-compatibility with it would be untestable (SURVEY §5.4, §7.4 item 8).
"""
from __future__ import annotations

import json
import os
import re
import threading
import time
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

STATE_FILE = "checkpoint"
PREFIX = "model.ckpt"
_DATA_SUFFIX = ".data-00000-of-00001"
_INDEX_SUFFIX = ".index"
_NP_DTYPES = {"float32": np.float32, "int64": np.int64, "int32": np.int32}


class CheckpointState:
    """Parsed ``checkpoint`` state file (``tf.train.get_checkpoint_state`` analogue)."""

    def __init__(self, model_checkpoint_path: str, all_model_checkpoint_paths: List[str]):
        self.model_checkpoint_path = model_checkpoint_path
        self.all_model_checkpoint_paths = all_model_checkpoint_paths


def _atomic_write(path: str, data: bytes) -> None:
    tmp = "%s.tmp.%d.%d" % (path, os.getpid(), threading.get_ident())
    with open(tmp, "wb") as f:
        f.write(data)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def get_checkpoint_state(checkpoint_dir: str) -> Optional[CheckpointState]:
    path = os.path.join(checkpoint_dir, STATE_FILE)
    try:
        with open(path, "r") as f:
            text = f.read()
    except OSError:
        return None
    latest = re.search(r'^model_checkpoint_path:\s*"(.*)"\s*$', text, re.M)
    if not latest:
        return None
    allp = re.findall(r'^all_model_checkpoint_paths:\s*"(.*)"\s*$', text, re.M)
    return CheckpointState(latest.group(1), allp)


def resolve_checkpoint_path(checkpoint_dir: str, state: CheckpointState) -> str:
    """Absolute vs relative handling of the reference (nn_eval.py:72-78)."""
    p = state.model_checkpoint_path
    return p if os.path.isabs(p) else os.path.join(checkpoint_dir, p)


def step_from_path(path: str) -> int:
    """``.../model.ckpt-1234`` -> 1234 (nn_eval.py:84)."""
    return int(path.split("/")[-1].split("-")[-1])


class Saver:
    """Save / restore named tensors under ``<dir>/model.ckpt-<step>``."""

    def __init__(self, max_to_keep: int = 5):
        self.max_to_keep = max_to_keep
        self._kept: List[str] = []
        self._lock = threading.Lock()

    def adopt(self, train_dir: str) -> None:
        """Continue the retention list of ``train_dir``'s state file, so ``max_to_keep`` also removes the checkpoints an
        earlier run wrote there."""
        st = get_checkpoint_state(train_dir)
        if st is not None:
            with self._lock:
                self._kept = [os.path.basename(p) for p in st.all_model_checkpoint_paths]

    # ---- write ------------------------------------------------------------
    def save(self, train_dir: str, tensors: Dict[str, torch.Tensor], global_step: int) -> str:
        os.makedirs(train_dir, exist_ok=True)
        prefix = os.path.join(train_dir, "%s-%d" % (PREFIX, int(global_step)))
        index: Dict[str, Dict] = {}
        blobs: List[bytes] = []
        off = 0
        named = dict(tensors)
        named["global_step"] = torch.tensor(int(global_step), dtype=torch.int64)
        for name in sorted(named):
            arr = named[name].detach().to("cpu").contiguous().numpy()
            if arr.dtype.name not in _NP_DTYPES:
                arr = arr.astype(np.float32)
            raw = arr.astype(arr.dtype.newbyteorder("<"), copy=False).tobytes()
            index[name] = {"dtype": arr.dtype.name, "shape": list(arr.shape), "offset": off, "nbytes": len(raw)}
            blobs.append(raw)
            off += len(raw)
        with self._lock:
            _atomic_write(prefix + _DATA_SUFFIX, b"".join(blobs))
            _atomic_write(prefix + _INDEX_SUFFIX, json.dumps(
                {"format": "dmnist-b200-ckpt-v1", "global_step": int(global_step), "saved_at": time.time(),
                 "tensors": index}, indent=1).encode())
            rel = os.path.basename(prefix)
            if rel in self._kept:
                self._kept.remove(rel)
            self._kept.append(rel)
            while len(self._kept) > self.max_to_keep:
                old = self._kept.pop(0)
                for suf in (_DATA_SUFFIX, _INDEX_SUFFIX):
                    try:
                        os.remove(os.path.join(train_dir, old + suf))
                    except OSError:
                        pass
            lines = ['model_checkpoint_path: "%s"' % rel]
            lines += ['all_model_checkpoint_paths: "%s"' % k for k in self._kept]
            # State file last: a reader that sees the new path always finds the data.
            _atomic_write(os.path.join(train_dir, STATE_FILE), ("\n".join(lines) + "\n").encode())
        return prefix

    # ---- read -------------------------------------------------------------
    @staticmethod
    def restore(prefix: str) -> Tuple[Dict[str, torch.Tensor], int]:
        with open(prefix + _INDEX_SUFFIX, "r") as f:
            meta = json.load(f)
        with open(prefix + _DATA_SUFFIX, "rb") as f:
            data = f.read()
        out: Dict[str, torch.Tensor] = {}
        for name, ent in meta["tensors"].items():
            dt = np.dtype(_NP_DTYPES[ent["dtype"]]).newbyteorder("<")
            arr = np.frombuffer(data, dtype=dt, count=int(np.prod(ent["shape"])) if ent["shape"] else 1,
                                offset=ent["offset"]).reshape(ent["shape"])
            out[name] = torch.from_numpy(np.array(arr, dtype=_NP_DTYPES[ent["dtype"]]))
        step = int(out.pop("global_step").item()) if "global_step" in out else int(meta["global_step"])
        return out, step

    @staticmethod
    def latest(checkpoint_dir: str) -> Optional[str]:
        st = get_checkpoint_state(checkpoint_dir)
        if st is None or not st.model_checkpoint_path:
            return None
        p = resolve_checkpoint_path(checkpoint_dir, st)
        return p if os.path.exists(p + _INDEX_SUFFIX) else None
