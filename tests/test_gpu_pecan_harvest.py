"""cPecan-mode recordings on the GPU (-m gpu): tests/golden/pecan_harvest.bin (a reference cPecan-mode bar() run recorded by
shim/cactus_pecan_harvest.c, scripts/make_golden_pecan_harvest.py) replayed through libbarb200's C ABI -- MUM anchors with
barb200_pecan_anchor_pairs_batch, posteriors with barb200_pecan_aligned_pairs_batch -- one end per call and all ends in one call,
on a single device and on a context over every visible device; every pair's anchor and triple hashes equal the reference's."""
import os
import subprocess
import sys

import pytest

import _reflib as R
import workload
from workload import pecan_replay as PR

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(R.ROOT, "tests", "golden", "pecan_harvest.bin")


@pytest.fixture(scope="module")
def ends():
    return workload.read_pecan_harvest(GOLDEN)


def _replay(ends, all_devices, settings):
    import cactus_b200
    ctx = PR.Context(cactus_b200.library_path(), all_devices=all_devices)
    try:
        s0 = ctx.device_stats()
        runs = {n: PR.replay(ctx, ends, n) for n in settings}
        s1 = ctx.device_stats()
    finally:
        ctx.close()
    return runs, (s1[0] - s0[0], s1[1] - s0[1])


def test_fixture_replays_bit_exact_on_one_device(ends):
    n_pairs = sum(len(e["pairs"]) for e in ends)
    runs, (hmm, mum) = _replay(ends, False, (1, 0))
    for n, r in runs.items():
        assert r["mismatches"] == [], n
        assert r["pairs"] == n_pairs and r["calls"] == (len(ends) if n == 1 else 1)
        assert r["anchor_calls"] > 0 and r["anchor_device_ms"] > 0 and r["cells"] > 0
    assert runs[1]["cells"] == runs[0]["cells"]
    assert len(hmm) == 1 and hmm[0] == 2 * n_pairs and mum[0] > 0


def test_fixture_replays_bit_exact_on_every_device(ends):
    import torch
    n_pairs = sum(len(e["pairs"]) for e in ends)
    runs, (hmm, mum) = _replay(ends, True, (0, 1))
    for n, r in runs.items():
        assert r["mismatches"] == [], n
        assert r["pairs"] == n_pairs
    assert len(hmm) == torch.cuda.device_count() and int(hmm.sum()) == 2 * n_pairs
    if len(hmm) >= 2:
        assert (hmm > 0).sum() > 1, hmm.tolist()


def test_replay_script_passes_its_parity_gate(tmp_path):
    out = tmp_path / "report.json"
    p = subprocess.run([sys.executable, os.path.join(R.ROOT, "scripts", "pecan_replay.py"), GOLDEN, "--json", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout + p.stderr
    assert "parity: every pair's anchors and triples equal the recording" in p.stdout
    import json
    rep = json.loads(out.read_text())
    assert rep["parity"] == "passed" and [s["ends_per_batch"] for s in rep["settings"]] == [1, 0]
    assert all(s["gcell_per_s"] > 0 for s in rep["settings"])
