#!/usr/bin/env python
"""Turn the compute times of cdf-mode runs into a straggler profile for ``--inject_straggler rank:profile:PATH``.

    python tools/straggler_profile.py OUT.npy MASTER_LOG [MASTER_LOG ...] [--with_master] [--absolute]

Each master log's last ``ELAPSED TIMES`` line (tools/benchmark.py ``extract_compute_times_no_master``; ``--with_master``
keeps the chief's own samples) gives (seconds, worker, iteration) samples.  By default the profile holds every sample's
excess over its run's median compute time, in microseconds and clipped at zero: replaying it adds the measured spread on
top of the replica's own compute instead of counting the baseline compute twice.  ``--absolute`` keeps the raw times.
"""
from __future__ import annotations

import os
import sys
from typing import Sequence

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from benchmark import extract_compute_times, extract_compute_times_no_master  # noqa: E402


def profile_from_logs(logs: Sequence[str], with_master: bool = False, absolute: bool = False) -> np.ndarray:
    """Delays in microseconds, the samples of every log concatenated."""
    out = []
    for path in logs:
        rows = extract_compute_times(path) if with_master else extract_compute_times_no_master(path)
        if not rows:
            raise ValueError("%s: no ELAPSED TIMES samples" % path)
        us = np.array([t for t, _w, _i in rows], dtype=np.float64) * 1e6
        if not absolute:
            us = np.maximum(us - np.median(us), 0.0)
        out.append(us)
    return np.concatenate(out)


def main(argv: Sequence[str]) -> int:
    args = [a for a in argv if not a.startswith("--")]
    if len(args) < 2:
        print(__doc__)
        return 2
    prof = profile_from_logs(args[1:], with_master="--with_master" in argv, absolute="--absolute" in argv)
    np.save(args[0], prof)
    q = np.quantile(prof, [0.5, 0.9, 0.99, 1.0])
    print("%s: %d samples; p50 %.1f us, p90 %.1f us, p99 %.1f us, max %.1f us" % ((args[0], prof.size) + tuple(q)))
    return 0


if __name__ == "__main__":
    sys.exit(main(sys.argv[1:]))
