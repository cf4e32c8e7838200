"""CPU tests of the non-convolution case table (tests/op_cases.py):
  * every case reaches the kernel variant it names (the host restatement of its entry point's dispatch);
  * the table as a whole reaches every variant: a variant no case reaches fails here, by name;
  * (tests/test_model_op_launches_cpu.py) every non-convolution launch the shipped models issue, and the post-op of every
    convolution, falls in a variant class of the table;
  * the GroupNorm inputs of the models stay within the mean/std range tests/test_op_cases_gpu.py asserts its bar over."""
import pathlib

import pytest
import torch

import op_cases as OC

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def classified():
    """(case, variant class, features) of every case, from the launch arguments built on host tensors"""
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    mp = pytest.MonkeyPatch()
    mp.setattr(L, "DRY_RUN", True)      # host tensors are accepted as operands; nothing is launched
    try:
        out = []
        for c in OC.CASES:
            t = OC.inputs(c, "cpu")
            o = {n: torch.empty(s, dtype=dt) for n, (s, dt) in OC.out_specs(c).items()}
            name, args = OC.launch(c, ops, t, o)
            cls, feats = OC.classify(name, OC.fields(name, args))
            out.append((c, cls, feats | OC.tags(c)))
        return out
    finally:
        mp.undo()


def test_case_ids_are_unique():
    ids = [c.id for c in OC.CASES]
    assert len(ids) == len(set(ids)), sorted(i for i in ids if ids.count(i) > 1)


def test_cases_reach_their_variant(classified):
    bad = [(c.id, c.want, cls) for c, cls, _ in classified if cls != c.want]
    assert not bad, "\n".join(f"{i}: wants {w}, reaches {g}" for i, w, g in bad)


def test_case_table_reaches_every_variant(classified):
    reached = {}
    for c, _, feats in classified:
        for f in feats:
            reached.setdefault(f, []).append(c.id)
    req = OC.required()
    print("\n[non-convolution kernel coverage] variant: cases reaching it")
    for r in req:
        print(f"  {r:40s} {len(reached.get(r, [])):3d}  {reached.get(r, ['-'])[0]}")
    missing = [r for r in req if r not in reached]
    assert not missing, f"variants no case of tests/op_cases.py reaches: {missing}"


def test_model_groupnorm_inputs_stay_near_zero_mean():
    """The largest per-group |mean| / std over every GroupNorm input of the oracle's source + driver passes at 256^2 and 512^2
    (seeded synthetic checkpoint, image-like frames) stays under op_cases.GN_MODEL_RATIO: the GPU sweep asserts the
    statistics producers' error bar up to twice that ratio (tests/test_op_cases_gpu.py::test_groupnorm_offset_data)."""
    import torch.nn.functional as F

    from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
    from emoportraits_b200.config import shipped_config
    from oracle import frames as FR
    from oracle import restatement as R

    orig, seen = F.group_norm, []

    def group_norm(x, G, *a, **kw):
        t = x.detach().double().reshape(x.shape[0], G, -1)
        std = t.std(-1, unbiased=False)
        seen.append(((t.mean(-1).abs() / std.clamp_min(1e-30))[std > 0].max().item(), tuple(x.shape)))
        return orig(x, G, *a, **kw)

    mp = pytest.MonkeyPatch()
    mp.setattr(R.F, "group_norm", group_norm)
    try:
        for size in (256, 512):
            cfg = shipped_config(size)
            sd, hsd = synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0)
            ocfg = R.config_from_state_dict(sd, size)
            with torch.no_grad():
                st = R.source_pass(sd, hsd, FR.frame(size, 41, "smooth"), ocfg)
                R.driver_pass(sd, hsd, st, FR.frame(size, 42, "smooth"), ocfg)
    finally:
        mp.undo()
    ratio, shape = max(seen)
    print(f"\n[GroupNorm inputs of stage 1 at 256^2 and 512^2] {len(seen)} normalisations, largest |mean| / std {ratio:.2f} "
          f"(input {shape}); asserted bound {OC.GN_MODEL_RATIO}")
    assert len(seen) > 100
    assert ratio < OC.GN_MODEL_RATIO, (ratio, shape)
