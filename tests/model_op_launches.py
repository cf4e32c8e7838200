"""Every non-convolution kernel launch the shipped models issue, recorded in EMO_DRY_RUN mode, and the launches of the wrapper
boundary, listed by hand.

A model launch is any C-ABI call of the configurations of model_conv_launches.CONFIGS except emo_conv_igemm (its own table,
tests/model_conv_launches.json) and the benchmark's L2 flushes.  The pose algebra's smoothing launches come from the stage-1
wrapper, not from the models: the smoothing cases of tests/op_cases.py cover them.  It is stored as
its entry point (`op`), every scalar argument or scalar descriptor field (`args`), the names of its non-NULL pointers (`ptrs`),
and the variant class and features op_cases.classify gives it.  Launches with equal records are one entry of the table, which
lists the configurations each came from.  tests/model_op_launches.json is the table of CONFIGS; tests/test_model_op_launches_cpu.py
checks that it is current and that every launch falls in a variant some case of tests/op_cases.py checks, and
tests/test_model_op_launches_gpu.py replays every entry against float64.  Regenerate it after a model change with

    python tests/model_op_launches.py --write

`python tests/model_op_launches.py CONFIG...` prints the table of the given configurations after "LAUNCHES ".

The wrappers (infer.InferenceWrapper, stage2.InferenceWrapper, video.drive_image_with_video, masks.FaceParsing /
modnet_get_mask) need a CUDA device, so their launches cannot be recorded here: BOUNDARY lists them, each with the line of code
that issues it, at the sizes the wrappers run.  tests/test_model_op_launches_gpu.py runs the wrappers live and fails on any
boundary launch whose class and argument pattern (`pattern`) no BOUNDARY entry has."""
from __future__ import annotations

import ctypes as C
import json
import os
import pathlib
import sys

ROOT = pathlib.Path(__file__).resolve().parents[1]
TABLE = pathlib.Path(__file__).resolve().parent / "model_op_launches.json"
sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent))

import model_conv_launches as MCL  # noqa: E402
import op_cases as OC  # noqa: E402

CONFIGS = MCL.CONFIGS
NOT_RECORDED = ("emo_conv_igemm", "emo_l2_flush", "emo_l2_flush_clean")
SIZE_ARGS = ("N", "H", "W", "Hin", "Win", "Hout", "Wout")   # what `pattern` leaves out


def launch_record(name: str, args) -> dict:
    """the record of one C-ABI call (pointer values excluded)"""
    f = OC.fields(name, args)
    ptr_names = OC.pointer_fields(name, args)
    cls, feats = OC.classify(name, f)
    return dict(op=name[4:], args={k: v for k, v in f.items() if k not in ptr_names}, ptrs=sorted(k for k in ptr_names if f[k]),
                cls=cls, features=sorted(feats))


def key(rec: dict) -> str:
    """the identity of a launch: its whole record"""
    return json.dumps({k: v for k, v in rec.items() if k not in ("configs", "site")}, sort_keys=True)


def pattern(rec: dict) -> str:
    """class and argument pattern of a launch: its record without the sizes (what the wrappers' live calls must match)"""
    return json.dumps(dict(op=rec["op"], cls=rec["cls"], ptrs=rec["ptrs"],
                           args={k: v for k, v in rec["args"].items() if k not in SIZE_ARGS}), sort_keys=True)


def record(config: str) -> list:
    """the records of every recorded C-ABI call of one configuration, in launch order (needs lib.DRY_RUN)"""
    recs = []

    def hook(name, *args):
        if name not in NOT_RECORDED:
            recs.append(launch_record(name, args))

    MCL.run(config, hook)
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


def load() -> list:
    """the committed table"""
    return json.loads(TABLE.read_text())


def dumps(rows) -> str:
    """one launch per line"""
    return "[\n" + ",\n".join(json.dumps(r, sort_keys=True) for r in rows) + "\n]\n"


# ------------------------------------------------------------------------------------------------------------------
# statistics producers: the longest run of fp32 additions one thread makes before its partial sum goes to an fp64 atomic or
# the final division, computed from the launch arguments as the host code sizes the grid
# ------------------------------------------------------------------------------------------------------------------
def serial_sum_length(rec: dict):
    """(producer, additions) of a statistics-producing launch, or None"""
    op, a, p = rec["op"], rec["args"], set(rec["ptrs"])
    if op == "gn_stats":
        c4n, N = a["C"] // 4, a["N"]
        chunks = min(max(1, a["S"] * c4n // 4096), max(1, (OC.SM_COUNT * 8) // N))
        rows_per_pass = 256 // min(c4n, 256)
        return "gn_stats", OC.cdiv(OC.cdiv(a["S"], chunks), rows_per_pass)
    if op == "global_avgpool":
        return "global_avgpool", a["S"]
    if op in ("upsample_trilinear", "avgpool") and "stats" in p:
        bx, fixed = OC.resample_grid(a, op == "avgpool")
        if not fixed:
            return f"{op} stats", 1
        per_n = a["D"] * a["H"] * a["W"] * (a["C"] // 4)
        per_n = per_n // (a["fd"] * a["fh"] * a["fw"]) if op == "avgpool" else per_n * a["fd"] * a["fh"] * a["fw"]
        return f"{op} stats", OC.cdiv(per_n, bx * 256)
    return None


# ------------------------------------------------------------------------------------------------------------------
# the wrapper boundary
# ------------------------------------------------------------------------------------------------------------------
# masks._LABELS_DEFAULT as the four class bit sets ops.parsing_masks passes
PARSING_LABEL_BITS = [425982, 409598, 262144, 65536]


def _b(op: str, site: str, **kw) -> dict:
    """a boundary launch: `kw` holds every argument of the entry point, pointers as True (set) or None (NULL)"""
    name = "emo_" + op
    args = [kw[k] for k in OC.POSITIONAL[name]]
    args = [(1 if v else 0) if k in OC.POSITIONAL_POINTERS else v for k, v in zip(OC.POSITIONAL[name], args)]
    rec = launch_record(name, args)
    rec["site"] = site
    return rec


def _boundary() -> list:
    rows = []
    conv = "emoportraits_b200/infer.py: return ops.u8_to_image(u8)"
    for n, (h, w) in [(1, (256, 256)), (32, (256, 256)), (1, (512, 512)), (32, (512, 512)), (1, (1080, 1920)), (1, (480, 640))]:
        rows.append(_b("u8_to_image", conv, x=True, N=n, H=h, W=w, C=3, out=True))
    prep = "emoportraits_b200/infer.py: t = ops.resize_bicubic(t, (s, s))"
    for hw in [(1080, 1920), (720, 1280), (480, 640), (200, 180)]:
        for s in (256, 512):
            rows.append(_b("resize_bicubic", prep, x=True, N=1, C=3, Hin=hw[0], Win=hw[1], Hout=s, Wout=s, out=True))
    to_u8 = [("emoportraits_b200/infer.py: ops.image_to_u8(img[i:i + 1], out=u8[i:i + 1])", 1, (256, 512)),
             ("emoportraits_b200/infer.py: host = ops.image_to_u8(img.detach().contiguous()).cpu().numpy()", 32, (256, 512)),
             ("emoportraits_b200/video.py: outs.extend(Image.fromarray(h) for h in ops.image_to_u8(img.contiguous()).cpu().numpy())",
              16, (256, 512)),
             ("emoportraits_b200/stage2.py: to_pil = lambda t: [Image.fromarray(h) for h in ops.image_to_u8(t.detach().contiguous().float()).cpu().numpy()]",
              16, (512, 1024))]
    for site, n, sizes in to_u8:
        for s in sizes:
            rows.append(_b("image_to_u8", site, x=True, N=n, C=3, H=s, W=s, out=True))
    rows.append(_b("composite", "emoportraits_b200/video.py: return ops.composite(img.contiguous().float(), mask.contiguous().float(), "
                   "bg.contiguous().float(), threshold)", img=True, mask=True, bg=True, N=16, C=3, H=512, W=512,
                   threshold=C.c_float(0.3), out=True))
    prep_site = "emoportraits_b200/masks.py: x512 = ops.parsing_prepare(x.to(self.device).float().contiguous(), self.mean, self.std, (512, 512))"
    masks_site = ("emoportraits_b200/masks.py: m = ops.parsing_masks(y.float().contiguous(), (h, w), (self.mask_labels, self.face_labels, "
                  "self.body_labels, self.cloth_labels))")
    for hw in [(512, 512), (1080, 1920)]:
        rows.append(_b("parsing_prepare", prep_site, x=True, N=1, C=3, Hin=hw[0], Win=hw[1], Hout=512, Wout=512, mean=True, std=True,
                       out=True))
        rows.append(_b("parsing_masks", masks_site, x=True, N=1, K=19, Hin=512, Win=512, Hout=hw[0], Wout=hw[1],
                       label_sets=PARSING_LABEL_BITS, out=True, labels=None))
    area_in = "emoportraits_b200/masks.py: im = ops.resize_area(img.float().contiguous(), (im_rh, im_rw), scale=2.0, shift=-1.0)"
    area_out = "emoportraits_b200/masks.py: return ops.resize_area(matte.float().contiguous(), (im_h, im_w))"
    # modnet_get_mask: (h, w) -> the reference size (512 on the short side, multiples of 32) -> back
    for (h, w), (rh, rw) in [((512, 512), (512, 512)), ((1080, 1920), (512, 896)), ((300, 400), (512, 672))]:
        rows.append(_b("resize_area", area_in, x=True, N=1, C=3, Hin=h, Win=w, Hout=rh, Wout=rw, scale=2.0, shift=-1.0, out=True))
        rows.append(_b("resize_area", area_out, x=True, N=1, C=1, Hin=rh, Win=rw, Hout=h, Wout=w, scale=1.0, shift=0.0, out=True))
    return rows


BOUNDARY = _boundary()


if __name__ == "__main__":
    os.environ["EMO_DRY_RUN"] = "1"   # before the package is imported: nothing is launched, host tensors stand in
    sys.path.insert(0, str(ROOT))
    args = sys.argv[1:]
    if args == ["--write"]:
        rows = table(CONFIGS)
        TABLE.write_text(dumps(rows))
        print(f"{TABLE.name}: {len(rows)} distinct launches")
    else:
        unknown = [a for a in args if a.split("-")[-1] not in MCL.PRECISIONS.get(a.split("-")[0], ())]
        if not args or unknown:
            sys.exit(f"usage: {sys.argv[0]} --write | CONFIG... (e.g. {' '.join(CONFIGS[:2])}); unknown: {unknown}")
        print("LAUNCHES " + json.dumps(table(args)))
