"""Every implicit-GEMM convolution (emo_conv_igemm) the shipped models launch, recorded in EMO_DRY_RUN mode.

A launch is stored as every scalar field of its emo_conv_desc, the names of the pointers it sets, the same for the
emo_apply_desc of its post-op (`post`), and the plan emo_conv_plan gives at 132 SMs (H100 SXM).  Launches with equal records
(pointers aside) are one entry of the table, which lists the configurations each came from.  tests/model_conv_launches.json is
the table of CONFIGS; tests/test_model_conv_launches_cpu.py checks that it is current and tests/test_model_conv_launches_gpu.py
replays every entry against float64.  Regenerate it after a model change with

    python tests/model_conv_launches.py --write

`python tests/model_conv_launches.py CONFIG...` prints the table of the given configurations after "LAUNCHES "."""
from __future__ import annotations

import ctypes as C
import json
import os
import pathlib
import sys

ROOT = pathlib.Path(__file__).resolve().parents[1]
TABLE = pathlib.Path(__file__).resolve().parent / "model_conv_launches.json"
SM_COUNT = 132   # H100 SXM

# stage 1: source pass + driver pass at S^2; stage 2: one forward at S^2 of a batch of B frames.  "srcfast" is stage 1 with
# the source pass on one fp16 plane (InferenceWrapper(source_precision="fast")); its driver pass is the exact mode's.  The
# tables list launches in order of first appearance: a configuration added at the end leaves the earlier entries in place.
CONFIGS = ("s1-256-exact", "s1-256-fast", "s1-512-exact", "s1-512-fast",
           "s2-512-b1-exact", "s2-512-b1-fast", "s2-1024-b4-exact", "s2-1024-b4-fast", "s2-1024-b16-exact", "s2-1024-b16-fast",
           "s1-256-srcfast", "s1-512-srcfast")
PRECISIONS = dict(s1=("exact", "fast", "srcfast"), s2=("exact", "fast"))   # the last field of a configuration, per stage


def _split(desc_type, d):
    """(scalar fields, names of the non-NULL pointer fields) of a ctypes descriptor"""
    scalars, ptrs = {}, []
    for name, t in desc_type._fields_:
        v = getattr(d, name)
        if t is C.c_void_p:
            if v:
                ptrs.append(name)
        else:
            scalars[name] = v
    return scalars, ptrs


def launch_record(L, lib, d) -> dict:
    """the record of one emo_conv_desc (pointer values excluded)"""
    conv, conv_ptrs = _split(L.ConvDesc, d)
    rec = dict(conv=conv, conv_ptrs=conv_ptrs, post=None, post_ptrs=None)
    if d.post:
        rec["post"], rec["post_ptrs"] = _split(L.ApplyDesc, C.cast(d.post, C.POINTER(L.ApplyDesc)).contents)
    info = L.ConvPlanInfo()
    rc = lib.emo_conv_plan(C.byref(d), SM_COUNT, C.byref(info))
    rec["rc"] = rc
    rec["err"] = lib.emo_last_error().decode() if rc else ""
    rec["plan"] = {f: getattr(info, f) for f, _ in info._fields_}
    return rec


def key(rec: dict) -> str:
    """the identity of a launch: its whole record"""
    return json.dumps({k: v for k, v in rec.items() if k != "configs"}, sort_keys=True)


def run(config: str, hook) -> None:
    """run the models of one configuration in EMO_DRY_RUN mode, calling hook(name, *args) before every C-ABI call"""
    import torch

    from emoportraits_b200 import lib as L

    assert L.DRY_RUN, "the models are recorded in EMO_DRY_RUN mode"
    launch = L.call

    def call(name, *args):
        hook(name, *args)
        return launch(name, *args)

    stage, size, *rest = config.split("-")
    precision = rest[-1]
    L.call = call
    try:
        torch.manual_seed(0)
        if stage == "s1":
            from emoportraits_b200.checkpoint import synthetic_head_pose_state_dict, synthetic_state_dict
            from emoportraits_b200.config import shipped_config
            from emoportraits_b200.infer import Model

            if precision == "srcfast":   # what InferenceWrapper(source_precision="fast") passes
                precision = dict(Model.PRESETS["exact"], **Model.SOURCE_FAST)
            cfg = shipped_config(int(size))
            model = Model(cfg, synthetic_state_dict(cfg, 0), synthetic_head_pose_state_dict(0), "cpu", precision=precision)
            x = torch.rand(1, 3, int(size), int(size))
            model.driver_pass(model.source_pass(x), x, mix=True)
        else:
            from emoportraits_b200.stage2 import Stage2Config, Stage2Model, synthetic_state_dict_s2

            cfg = Stage2Config(output_size=int(size))
            model = Stage2Model(cfg, synthetic_state_dict_s2(cfg, 0), "cpu", precision=precision)
            model.forward(torch.rand(int(rest[0][1:]), 3, 512, 512))
    finally:
        L.call = launch


def record(config: str) -> list:
    """the records of every emo_conv_igemm call of one configuration, in launch order (needs lib.DRY_RUN)"""
    from emoportraits_b200 import lib as L

    lib = L.load()
    recs = []

    def hook(name, *args):
        if name == "emo_conv_igemm":
            recs.append(launch_record(L, lib, args[0]._obj))

    run(config, hook)
    return recs


def table(configs) -> list:
    """the distinct launches of `configs`, in order of first appearance, each with the configurations it came from"""
    rows = {}
    for cfg in configs:
        for rec in record(cfg):
            row = rows.setdefault(key(rec), dict(rec, configs=[]))
            if cfg not in row["configs"]:
                row["configs"].append(cfg)
    return list(rows.values())


def out_elems(rec: dict) -> int:
    """elements of a launch's convolution output"""
    d = rec["conv"]
    return d["N"] * d["Dout"] * d["Hout"] * d["Wout"] * d["Cout"]


def load() -> list:
    """the committed table"""
    return json.loads(TABLE.read_text())


def dumps(rows) -> str:
    """one launch per line"""
    return "[\n" + ",\n".join(json.dumps(r, sort_keys=True) for r in rows) + "\n]\n"


if __name__ == "__main__":
    os.environ["EMO_DRY_RUN"] = "1"   # before the package is imported: nothing is launched, host tensors stand in
    sys.path.insert(0, str(ROOT))
    args = sys.argv[1:]
    if args == ["--write"]:
        rows = table(CONFIGS)
        TABLE.write_text(dumps(rows))
        print(f"{TABLE.name}: {len(rows)} distinct launches")
    else:
        unknown = [a for a in args if a.split("-")[-1] not in PRECISIONS.get(a.split("-")[0], ())]
        if not args or unknown:
            sys.exit(f"usage: {sys.argv[0]} --write | CONFIG... (e.g. {' '.join(CONFIGS[:2])}); unknown: {unknown}")
        print("LAUNCHES " + json.dumps(table(args)))
