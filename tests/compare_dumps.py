"""Diagnostic (not a test): compare two directories written by `bench.py --dump-outputs` (energy.npy, forces.npy,
stress.npy) and print |dE| / N, max |dF| and max |dsigma| as one JSON line.

    python tests/compare_dumps.py DIR_A DIR_B
"""
import json
import os
import sys

import numpy as np


def main():
    a, b = sys.argv[1], sys.argv[2]
    e, f, s = ([np.load(os.path.join(d, n + ".npy")).astype(np.float64) for d in (a, b)]
               for n in ("energy", "forces", "stress"))
    n = len(f[0])
    print(json.dumps({"a": a, "b": b, "atoms": n, "dE_per_atom": float(abs(e[0][0] - e[1][0]) / n),
                      "max_dF": float(np.abs(f[0] - f[1]).max()), "max_dS": float(np.abs(s[0] - s[1]).max())}))


if __name__ == "__main__":
    main()
