"""CPU checks of the table of model non-convolution launches (tests/model_op_launches.py, replayed on the GPU by
tests/test_model_op_launches_gpu.py):
  * recorded afresh in EMO_DRY_RUN mode, the launches of the twelve configurations (stage 1 at 256^2 and 512^2 in exact
    mode, fast mode and with the fast source pass; stage 2 at 512^2 batch 1 and 1024^2 batch 4 and 16, each in exact and fast
    mode) equal the committed table, so that a model change fails here until the table is regenerated;
  * every launch, and the post-op of every model convolution (tests/model_conv_launches.json), falls in a variant class that a
    case of tests/op_cases.py checks against float64;
  * the wrapper-boundary list names lines that exist, and the mask helpers, run on host tensors, issue exactly its launches.
Per configuration it prints the number of distinct launches, the largest launch per entry point and the longest per-thread
run of fp32 additions of each statistics producer."""
import ctypes as C
import json
import math
import os
import pathlib
import subprocess
import sys

import pytest
import torch

import model_conv_launches as MCL
import model_op_launches as MOL
import op_cases as OC

ROOT = pathlib.Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def fresh():
    env = dict(os.environ, EMO_DRY_RUN="1")
    r = subprocess.run([sys.executable, str(ROOT / "tests" / "model_op_launches.py"), *MOL.CONFIGS], env=env,
                       capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout + r.stderr
    return json.loads(r.stdout.split("LAUNCHES ", 1)[1])


SIZE_DIMS = ("N", "D", "H", "W", "C", "S", "n", "M", "K", "Dout", "Hout", "Wout", "Cout")


def _elems(rec) -> int:
    """a launch's size, to pick the largest per entry point: the product of its shape arguments"""
    return math.prod(v for k, v in rec["args"].items() if k in SIZE_DIMS)


def test_committed_table_is_current(fresh):
    committed = MOL.load()
    gone = {MOL.key(r) for r in committed} - {MOL.key(r) for r in fresh}
    new = {MOL.key(r) for r in fresh} - {MOL.key(r) for r in committed}
    print(f"\n[model op launches] {len(fresh)} distinct launches")
    for cfg in MOL.CONFIGS:
        rows = [r for r in fresh if cfg in r["configs"]]
        print(f"  {cfg:18s} {len(rows):4d} distinct launches")
        largest = {}
        for r in rows:
            if r["op"] not in largest or _elems(r) > _elems(largest[r["op"]]):
                largest[r["op"]] = r
        for op, r in sorted(largest.items()):
            print(f"      largest {op:22s} {json.dumps(r['args'], sort_keys=True)}")
        serial = {}
        for r in rows:
            s = MOL.serial_sum_length(r)
            if s is not None and s[1] > serial.get(s[0], (0, None))[0]:
                serial[s[0]] = (s[1], r)
        for prod, (n, r) in sorted(serial.items()):
            print(f"      longest fp32 serial sum {prod:26s} {n:6d} additions  {json.dumps(r['args'], sort_keys=True)}")
    assert not gone and not new and fresh == committed, (
        f"tests/model_op_launches.json is stale ({len(new)} new launches, {len(gone)} gone, or other configurations): "
        "regenerate it with `python tests/model_op_launches.py --write`")


def test_table_covers_every_configuration(fresh):
    seen = {c for r in fresh for c in r["configs"]}
    assert seen == set(MOL.CONFIGS), sorted(set(MOL.CONFIGS) - seen)
    assert not {r["op"] for r in fresh} & {n[4:] for n in MOL.NOT_RECORDED}


def _post_class(rec):
    """variant class of a convolution's post-op (an emo_apply_desc) from its record in the conv table"""
    from emoportraits_b200 import lib as L

    ptrs = {f for f, t in L.ApplyDesc._fields_ if t is C.c_void_p}
    f = dict(rec["post"], **{p: (1 if p in rec["post_ptrs"] else 0) for p in ptrs})
    return OC.classify("emo_apply", f)[0]


def test_every_launch_falls_in_a_checked_variant(fresh):
    """every recorded launch, and every conv post-op, is in a variant class some case of tests/op_cases.py reaches; this
    covers fast mode and stage 2 at batch 4 and 16"""
    covered = {c.want for c in OC.CASES}
    classes = {}
    for r in fresh:
        assert r["op"] not in OC.NOT_IN_TABLE, r["op"]
        for cfg in r["configs"]:
            classes.setdefault(cfg, {}).setdefault(r["cls"], 0)
            classes[cfg][r["cls"]] += 1
    for r in MCL.load():
        if r["post"]:
            cls = "conv post-op: " + _post_class(r)
            for cfg in r["configs"]:
                classes.setdefault(cfg, {}).setdefault(cls, 0)
                classes[cfg][cls] += 1
    uncovered = set()
    for cfg in MOL.CONFIGS:
        print(f"\n[{cfg} non-convolution launches: distinct launches per variant class]")
        for cls, n in sorted(classes[cfg].items()):
            base = cls.split(": ", 1)[-1]
            print(f"  {n:4d}  {cls}{'' if base in covered else '   <- no case'}")
            if base not in covered:
                uncovered.add(cls)
    assert not uncovered, f"model launches in variants no case of tests/op_cases.py checks: {sorted(uncovered)}"


def test_boundary_sites_are_lines_of_the_wrappers():
    for r in MOL.BOUNDARY:
        path, line = r["site"].split(": ", 1)
        assert line in (ROOT / path).read_text(), r["site"]
    assert {r["op"] for r in MOL.BOUNDARY} == {"u8_to_image", "image_to_u8", "resize_bicubic", "composite", "parsing_prepare",
                                                "parsing_masks", "resize_area"}


def test_mask_helpers_issue_the_boundary_launches():
    """FaceParsing.forward and modnet_get_mask on host tensors (EMO_DRY_RUN: nothing is launched) at 512^2, 1920x1080 and
    300x400: every launch is a BOUNDARY entry, sizes included"""
    from emoportraits_b200 import lib as L
    from emoportraits_b200.masks import FaceParsing, modnet_get_mask
    from oracle.stub_nets import StubBiSeNet, StubMODNet

    listed = {MOL.key(r) for r in MOL.BOUNDARY}
    recs = []
    launch = L.call

    def call(name, *args):
        recs.append(MOL.launch_record(name, args))
        return launch(name, *args)

    mp = pytest.MonkeyPatch()
    mp.setattr(L, "DRY_RUN", True)
    mp.setattr(L, "call", call)
    try:
        fp = FaceParsing(None, device="cpu", net=StubBiSeNet())
        for h, w in ((512, 512), (1080, 1920)):
            fp.forward(torch.rand(1, 3, h, w))
        for h, w in ((512, 512), (1080, 1920), (300, 400)):
            modnet_get_mask(StubMODNet(), torch.rand(1, 3, h, w))
    finally:
        mp.undo()
    assert len(recs) == 10, [r["op"] for r in recs]
    missing = [r for r in recs if MOL.key(r) not in listed]
    assert not missing, missing
