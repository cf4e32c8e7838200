"""CPU checks of the table of model convolution launches (tests/model_conv_launches.py, replayed on the GPU by
tests/test_model_conv_launches_gpu.py):
  * recorded afresh in EMO_DRY_RUN mode, the launches of the twelve configurations (model_conv_launches.CONFIGS) equal the
    committed table, so that a model change fails here until the table is regenerated;
  * no launch is refused and every launch plans, at 132 SMs, in a class that a GPU case of the same dimension (2-D or 3-D)
    sweeps (tests/conv_plan_cases.py and the fast-mode case lists);
  * the replay's float64 references (a sum over taps of shifted-activation matrix products, and its sub-pixel form) equal
    torch's float64 convolutions."""
import json
import os
import pathlib
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import conv_plan_cases as CP
import model_conv_launches as MCL

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def fresh():
    env = dict(os.environ, EMO_DRY_RUN="1")
    r = subprocess.run([sys.executable, str(ROOT / "tests" / "model_conv_launches.py"), *MCL.CONFIGS], env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.split("LAUNCHES ", 1)[1])


def test_committed_table_is_current(fresh):
    committed = MCL.load()
    gone = {MCL.key(r) for r in committed} - {MCL.key(r) for r in fresh}
    new = {MCL.key(r) for r in fresh} - {MCL.key(r) for r in committed}
    print(f"\n[model conv launches] {len(fresh)} distinct launches")
    for cfg in MCL.CONFIGS:
        rows = [r for r in fresh if cfg in r["configs"]]
        biggest = max(rows, key=lambda r: MCL.out_elems(r))
        print(f"  {cfg:18s} {len(rows):4d} distinct launches, largest output {MCL.out_elems(biggest):,} elements "
              f"({4 * MCL.out_elems(biggest) / 2 ** 30:.2f} GiB fp32)")
    assert not gone and not new and fresh == committed, (
        f"tests/model_conv_launches.json is stale ({len(new)} new launches, {len(gone)} gone, or other configurations): "
        "regenerate it with `python tests/model_conv_launches.py --write`")


def _swept_classes():
    import test_fast_decoder_gpu as TD
    import test_fast_source_gpu as TF
    import test_fast_stage2_gpu as TS

    return ({c.want for c in CP.CASES} | {w for w, _ in TD.CASES} | {w for w, _ in TS.CASES} | {w for w, _ in TF.CASES}
            | {TF.DEPTH_CASE[0]})


def test_every_launch_plans_in_a_swept_class(fresh):
    """a class is "<kernel> BN<n> <loop> <finish>", with " 3-D" for inputs of depth > 1: a 2-D case does not sweep a 3-D
    launch's depth halo, padding and tiles, nor a 3-D case a 2-D launch's"""
    from emoportraits_b200 import lib as L

    refused = [(r["conv"], r["err"]) for r in fresh if r["rc"] != 0]
    assert not refused, refused
    swept = _swept_classes()
    classes = {}
    for r in fresh:
        cls = CP.plan_class(L.ConvPlanInfo(**r["plan"]), r["conv"]["Din"])
        classes.setdefault(cls, []).append(r)
    print(f"\n[model conv launches] {len(classes)} plan classes at {MCL.SM_COUNT} SMs")
    for cls, rows in sorted(classes.items()):
        print(f"  {cls:40s} {len(rows):4d}")
    unswept = sorted(set(classes) - swept)
    assert not unswept, f"model launches in plan classes no GPU case sweeps: {unswept}"


def test_reference_convolutions_match_torch():
    import test_model_conv_launches_gpu as TG
    from emoportraits_b200 import ops

    g = torch.Generator().manual_seed(5)
    for (D, H, W), k, s, p in [((1, 9, 11), (1, 3, 3), (1, 1, 1), (0, 1, 1)), ((1, 10, 13), (1, 4, 4), (1, 2, 2), (0, 1, 1)),
                               ((1, 8, 8), (1, 7, 1), (1, 1, 1), (0, 3, 0)), ((4, 6, 7), (3, 3, 3), (1, 1, 1), (1, 1, 1)),
                               ((5, 7, 6), (3, 3, 3), (2, 2, 2), (1, 1, 1)), ((3, 5, 5), (1, 1, 1), (1, 2, 2), (0, 0, 0))]:
        x = torch.randn(D, H, W, 6, generator=g, dtype=torch.float64)
        w = torch.randn(5, 6, *k, generator=g, dtype=torch.float64)
        want = F.conv3d(x.permute(3, 0, 1, 2)[None], w, stride=s, padding=p)[0].permute(1, 2, 3, 0)
        got = TG.conv_cl(x, w.permute(2, 3, 4, 1, 0), s, p)
        assert torch.allclose(got, want, rtol=0, atol=1e-12), (k, s, p)
    x = torch.randn(1, 5, 7, 6, generator=g, dtype=torch.float64)
    w = torch.randn(4, 6, 3, 3, generator=g)
    want = F.conv2d(F.interpolate(x.permute(0, 3, 1, 2), scale_factor=2, mode="nearest"), w.double(), padding=1).permute(0, 2, 3, 1)
    got = TG.upconv_cl(x, ops.fold_upconv_weight(w).double().transpose(3, 4))
    assert torch.allclose(got, want, rtol=0, atol=1e-5)     # the folded taps are fp32 sums
