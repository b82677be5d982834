"""The fp64 Kabsch rotation on the CPU: the bounds of tests/kabsch_check.py on the whole case table, for fp64 numpy
against the 50-digit reference, for every planted mutation of the restatement, and for the real `kabsch_rotation`
(csrc/ransac_dev.cuh, __host__ __device__) built into a small host program with nvcc."""
import os
import shutil
import subprocess

import numpy as np
import pytest

from tests import kabsch_check as kc
from tests.common import ROOT

CSRC = os.path.join(ROOT, "mickey_b200", "csrc")


@pytest.fixture(scope="module")
def table():
    T = kc.case_table()
    return T, {k: kc.Ref(v) for k, v in T.items()}


def _report(label, res):
    print(f"\n[{label}] max(err / bound) per class: " +
          ", ".join(f"{k} {w:.2g}" for k, (w, _) in res.items()))


def test_restatement_is_within_the_bounds(table):
    T, refs = table
    res = kc.per_class(T, kc.kabsch_np, refs)
    _report("restatement", res)
    bad = {k: w for k, (w, _) in res.items() if not w <= 1.0}
    assert not bad, bad


@pytest.mark.parametrize("mutation", [m for m in kc.MUTATIONS if m != "no_reorth"])
def test_planted_mutations_are_rejected(table, mutation):
    T, refs = table
    res = kc.per_class(T, lambda H: kc.kabsch_np(H, mutation), refs)
    rejected = sorted(k for k, (w, _) in res.items() if not w <= 1.0)
    print(f"\n[{mutation}] rejected by {len(rejected)} classes: {', '.join(rejected)}")
    assert rejected, mutation


def test_reorthogonalisation_is_redundant_after_the_sweep(table):
    """Dropping the re-orthogonalisation of u_2 cannot be rejected.  A pair is rotated whenever |cos| > 1e-15 and the
    sweep stops once every pair measured below 1e-14 at the start of a sweep; the rotations of that last sweep leave
    the pairs far closer to orthogonal than that (the convergence is quadratic), so u_2 is already orthogonal to u_1
    within a few u.  The mutation is kept to show that: it moves no entry of R by more than 8 u on the table."""
    T, _ = table
    for name, H in T.items():
        a, b = kc.kabsch_np(H), kc.kabsch_np(H, "no_reorth")
        fin = np.isfinite(a).all((1, 2))
        assert np.array_equal(np.isnan(a), np.isnan(b)), name
        if fin.any():
            assert float(np.abs(a - b)[fin].max()) <= 8 * kc.U64, name


HARNESS = r"""
#include <cstdio>
#include <vector>
#include "ransac_dev.cuh"
int main(int argc, char** argv) {
  FILE* f = fopen(argv[1], "rb");
  std::vector<double> H;
  double v[9];
  while (fread(v, sizeof(double), 9, f) == 9) H.insert(H.end(), v, v + 9);
  fclose(f);
  std::vector<double> R(H.size());
  for (size_t i = 0; i < H.size(); i += 9) mk::kabsch_rotation(&H[i], &R[i]);
  FILE* g = fopen(argv[2], "wb");
  fwrite(R.data(), sizeof(double), R.size(), g);
  fclose(g);
  return 0;
}
"""


@pytest.fixture(scope="module")
def host_kabsch(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    d = tmp_path_factory.mktemp("kabsch_host")
    src, exe = d / "kabsch_host.cu", d / "kabsch_host"
    src.write_text(HARNESS)
    # host code without FMA contraction: the same operation order as the numpy restatement
    subprocess.run([nvcc, "-std=c++17", "-O2", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-ffp-contract=off",
                    "-I", CSRC, "-o", str(exe), str(src)], check=True, capture_output=True, timeout=600)

    def run(H):
        H = np.ascontiguousarray(np.asarray(H, dtype=np.float64).reshape(-1, 9))
        H.tofile(d / "H.bin")
        subprocess.run([str(exe), str(d / "H.bin"), str(d / "R.bin")], check=True, timeout=120)
        return np.fromfile(d / "R.bin", dtype=np.float64).reshape(-1, 3, 3)
    return run


def test_host_build_of_kabsch_rotation_is_within_the_bounds(table, host_kabsch):
    """The real function (compiled for the host) on the whole table, scale and non-finite classes included."""
    T, refs = table
    res = kc.per_class(T, host_kabsch, refs)
    _report("kabsch_rotation, host build", res)
    bad = {k: w for k, (w, _) in res.items() if not w <= 1.0}
    assert not bad, bad


def test_host_build_equals_the_restatement(table, host_kabsch):
    """Without FMA contraction the restatement is the same arithmetic: bit-identical R (NaN where H is not finite)."""
    T, _ = table
    for name, H in T.items():
        a, b = host_kabsch(H), kc.kabsch_np(H)
        assert np.array_equal(a, b, equal_nan=True), (name, float(np.nanmax(np.abs(a - b))))
