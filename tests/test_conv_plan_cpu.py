"""CPU test of the implicit-GEMM convolution's launch planner (emo_conv_plan, the planning half of emo_conv_igemm):
  * every case of tests/conv_plan_cases.py reaches the plan class it names at 132 SMs (H100 SXM);
  * the case table as a whole reaches every configuration of the kernel (instantiations, wgmma N widths, main loops,
    split-K finish paths, ragged boxes, padded / odd Cout, both statistics branches, ...): a later change of the planner's
    heuristics that leaves a configuration unchecked by tests/test_conv_plan_gpu.py fails here, naming it;
  * every convolution the shipped models issue (stage 1 at 256 and 512, stage 2 at 512 and 1024: recorded in EMO_DRY_RUN
    mode) passes the planner's checks and falls in a plan class the case table covers with a case of its dimension (a
    " 3-D" class for inputs of depth > 1)."""
import json
import os
import pathlib
import subprocess
import sys

import pytest
import torch

import conv_plan_cases as CP

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def plans():
    """(case, emo_conv_plan_info at 132 SMs) of every case, planned from host tensors (the planner reads no operand)"""
    from emoportraits_b200 import lib as L
    from emoportraits_b200 import ops

    mp = pytest.MonkeyPatch()
    mp.setattr(L, "DRY_RUN", True)      # host tensors are accepted as operands; nothing is launched
    try:
        out = []
        for c in CP.CASES:
            x, w, b, res, pa = CP.make(c, "cpu")
            st = torch.zeros((c.N, c.G, 2), dtype=torch.float64) if (c.stats or c.post) else None
            a, pw, kw = CP.conv_args(c, ops, x, w, b, res, pa, stats=st)
            out.append((c, ops.conv_plan(a, pw, sm_count=CP.SM_COUNT, **kw)))
        return out
    finally:
        mp.undo()


def test_header_enums_match_the_binding():
    import re

    from emoportraits_b200 import lib as L

    hdr = (ROOT / "include" / "emoportraits_b200.h").read_text()
    kern = dict((int(v), n) for n, v in re.findall(r"EMO_CONV_KERNEL_(\w+) = (\d+)", hdr))
    fin = dict((int(v), n) for n, v in re.findall(r"EMO_CONV_FINISH_(\w+) = (\d+)", hdr))
    assert sorted(kern) == list(range(len(L.CONV_KERNELS))) and sorted(fin) == list(range(len(L.CONV_FINISH)))
    assert [n.lower().replace("_", "+") for _, n in sorted(fin.items())] == list(L.CONV_FINISH)
    for i, name in enumerate(L.CONV_KERNELS):      # "conv<64,2>" <-> BF16X2_KC64 ...
        form = {"conv": "BF16X" + name[-2], "f16": "F16", "ps": "UPCONV"}[name.split("<")[0]]
        assert kern[i] == f"{form}_KC{name.split('<')[1][:2]}", (i, name, kern[i])


def test_cases_reach_their_plan_class(plans):
    bad = [(c.id, c.want, CP.plan_class(p, CP.depth(c))) for c, p in plans if CP.plan_class(p, CP.depth(c)) != c.want]
    assert not bad, "\n".join(f"{i}: wants {w}, plans {g}" for i, w, g in bad)


def _features(c, p):
    """the configurations one planned case exercises"""
    from emoportraits_b200 import lib as L

    kern = L.CONV_KERNELS[p.kernel]
    Do, Ho, Wo = CP.out_shape(c)
    gD, gH, gW = (1, c.sp[-2], c.sp[-1]) if c.upconv else (Do, Ho, Wo)
    split = p.ksplit > 1
    ragged = gW % p.tw != 0 or gH % p.th != 0 or gD % p.td != 0
    f = {f"kernel {kern}", f"{'fp16' if p.fp16 else 'bf16'} BN{p.BN}"}
    if p.yreuse:
        f.add(f"row reuse sa={p.sa}")
        f.add("row reuse in the sub-pixel kernel" if c.upconv else "row reuse in a plain kernel")
        if p.KC == 32:
            f.add(f"row reuse KC=32 {'fp16' if p.fp16 else f'NP={p.NP}'}")
    else:
        if p.td > 1:
            f.add("per-tap loop, 3-D box (td > 1)")
        if c.stride == 2:
            f.add(f"per-tap loop, stride 2, {len(c.sp)}-D")
    if split:
        f.add(f"split-K finish {L.CONV_FINISH[p.finish]}")
    if p.m_tiles * p.n_tiles * p.ksplit > p.grid:
        f.add(f"items > grid, {'row reuse' if p.yreuse else 'per-tap'} loop")
    if ragged:
        f.add(f"ragged box, {kern}")
    cout_pad = ((c.Cout + 15) // 16) * 16
    if c.Cout < cout_pad:
        f.add("Cout < Cout_pad")
    if c.Cout % 2:
        f.add("odd Cout (scalar final phase)")
    if c.Cout < 16:
        f.add("Cout < 16")
    if c.stats and not split:
        f.add("tile stats per group" if p.BN % (c.Cout // c.G) == 0 else "tile stats per column")
    for opt in ("out_nchw", "post_add"):
        if getattr(c, opt):
            f.add(f"{opt} {'split-K' if split else 'un-split'}")
    if c.res_shift:
        f.add(f"res_shift=1, {'ragged' if ragged else 'exact'} box")
    taps = 4 if c.upconv else (c.k ** len(c.sp) if len(c.sp) == 3 else c.k * c.k)
    if not split and (taps * c.Cin // p.KC) % p.flush:
        f.add("flush does not divide the k-steps")
    if c.acc:
        f.add("explicit acc_chunk_mmas")
    if c.N > 1 and c.stats:
        f.add("batch N > 1 with statistics")
    return f


def _required():
    from emoportraits_b200 import lib as L

    req = [f"kernel {k}" for k in L.CONV_KERNELS]
    req += [f"{t} BN{bn}" for t in ("bf16", "fp16") for bn in range(16, 129, 16)]
    req += ["row reuse sa=2", "row reuse sa=3", "row reuse KC=32 NP=2", "row reuse KC=32 NP=3", "row reuse KC=32 fp16",
            "row reuse in the sub-pixel kernel", "row reuse in a plain kernel", "per-tap loop, 3-D box (td > 1)",
            "per-tap loop, stride 2, 2-D", "per-tap loop, stride 2, 3-D"]
    req += [f"split-K finish {f}" for f in ("finalize", "post", "finalize+apply")]
    req += ["items > grid, row reuse loop", "items > grid, per-tap loop"]
    req += [f"ragged box, {k}" for k in L.CONV_KERNELS]
    req += ["Cout < Cout_pad", "odd Cout (scalar final phase)", "Cout < 16", "tile stats per group", "tile stats per column"]
    req += [f"{o} {s}" for o in ("out_nchw", "post_add") for s in ("un-split", "split-K")]
    req += ["res_shift=1, ragged box", "res_shift=1, exact box", "flush does not divide the k-steps", "explicit acc_chunk_mmas",
            "batch N > 1 with statistics"]
    return req


def test_case_table_reaches_every_configuration(plans):
    reached = {}
    for c, p in plans:
        for f in _features(c, p):
            reached.setdefault(f, []).append(c.id)
    req = _required()
    print("\n[conv plan coverage at 132 SMs] configuration: cases reaching it")
    for r in req:
        print(f"  {r:40s} {len(reached.get(r, [])):3d}  {reached.get(r, ['-'])[0]}")
    missing = [r for r in req if r not in reached]
    assert not missing, f"configurations no case of tests/conv_plan_cases.py reaches: {missing}"


def _old_key(rec):
    """the shape key this test used to file launches under: it left out res_shift, pads, strides other than sh, the operand
    planes and which optional pointers are set, so launches differing only there overwrote each other"""
    d = rec["conv"]
    return "%dx%dx%dx%dx%d->%d k%d%d%d s%d%s%s" % (d["N"], d["Din"], d["Hin"], d["Win"], d["Cin"], d["Cout"], d["kd"], d["kh"],
                                               d["kw"], d["sh"], " up2" if d["upconv"] else "", " post" if rec["post"] else "")


@pytest.mark.parametrize("model", ["s1-256", "s1-512", "s2-512", "s2-1024"])
def test_model_layers_fall_in_swept_plan_classes(model):
    """every distinct launch (tests/model_conv_launches.py's full record) of the exact-mode model; stage 2 at batch 1"""
    from emoportraits_b200 import lib as L

    config = model + ("-exact" if model.startswith("s1") else "-b1-exact")
    env = dict(os.environ, EMO_DRY_RUN="1")
    r = subprocess.run([sys.executable, str(ROOT / "tests" / "model_conv_launches.py"), config], env=env, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout + r.stderr
    rows = json.loads(r.stdout.split("LAUNCHES ", 1)[1])
    assert rows, "no emo_conv_igemm call recorded"
    refused = [(_old_key(v), v["err"]) for v in rows if v["rc"] != 0]
    assert not refused, refused
    swept = {c.want for c in CP.CASES}
    old = {_old_key(v) for v in rows}
    print(f"\n[{model} conv layers: plan class at 132 SMs] {len(rows)} distinct launches; the shape key alone would merge "
          f"{len(rows) - len(old)} of them into others")
    unswept = []
    for v in rows:
        d = v["conv"]
        info = L.ConvPlanInfo(**v["plan"])
        cls = CP.plan_class(info, d["Din"])
        opts = " ".join(sorted(set(v["conv_ptrs"]) - {"a_hi", "a_lo", "a_lo2", "w_hi", "w_lo", "w_lo2", "out", "splitk_ws"}))
        name = f"{_old_key(v)} p{d['ph']}{d['pw']} rs{d['res_shift']} act{d['act']} [{opts}]"
        print(f"  {name:90s} {cls:36s} ksplit {info.ksplit:2d} grid {info.grid:3d}")
        if cls not in swept:
            unswept.append((name, cls))
    assert not unswept, f"model layers in plan classes no case of tests/conv_plan_cases.py checks: {unswept}"
