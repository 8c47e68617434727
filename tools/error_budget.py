#!/usr/bin/env python
"""Error budget of the head MLP precision modes on the CPU oracle (no GPU needed).

Emulates, one site at a time, the roundings the wgmma modes introduce -- 16-bit grid tables, 16-bit A operands
(activations), 16-bit W operands (weights), per layer -- inside oracle/render.py's field query and reports the max-abs RGB
error of the rendered frame against the untouched fp32 oracle.  This is how the "robust" mode was chosen (DESIGN.md
"precision"): the site that dominates gets the hi/lo split, the others stay single 16-bit images.

    python tools/error_budget.py [--size 64] [--gain 4] [--ds 1] [--fold-only]

The first four lines compare k_head_v2's fp16 and robust modes with sigma L2's geo rows computed as their own layer (parent)
and folded into color L0 (DESIGN.md §6).
"""
import argparse
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from genefaceplusplus_b200 import scene as scn  # noqa: E402
from helpers import lively_state, parity_report  # noqa: E402
from oracle import ops  # noqa: E402
from oracle.render import OracleModel  # noqa: E402

LAYERS = ["amb0", "amb1", "amb2", "sig0", "sig1", "sig2", "col0", "col1"]


def r16(x, kind):
    if kind == "fp16":
        return x.half().float()
    if kind == "bf16":
        return x.bfloat16().float()
    raise ValueError(kind)


def split(x, kind):
    hi = r16(x, kind)
    return hi, r16(x - hi, kind)


class Emu:
    """linear(x, w) hook: per-layer operand treatment.  mode per layer: (a_mode, w_mode), each in
    {"f32", "x1" (one 16-bit image), "x2" (hi + lo images)}; products accumulate in fp32 (tensor-core behaviour).

    fold: the geo rows of sigma L2 folded into color L0 as k_head_v2 runs them -- sigma L2 computes only its sigma row and
    passes sigma L1's output through as "geo"; color L0's geo columns become W_fold = W_c0[:, 16:144] . W_s2[1:129, :]
    (double, then fp32, then the layer's W rounding), so h_s1 and W_fold are the only roundings on the geo path."""

    def __init__(self, state, kind, cfg, fold=False):
        self.kind = kind
        self.by_id = {}
        names = [f"ambient_net.net.{i}.weight" for i in range(3)] + [f"sigma_net.net.{i}.weight" for i in range(3)] + \
                [f"color_net.net.{i}.weight" for i in range(2)]
        self.names = dict(zip(names, LAYERS))
        self.cfg = cfg
        self.state = state
        self.fold = fold

    def bind(self, orc):
        for k, lay in self.names.items():
            self.by_id[id(orc.st[k])] = lay
        self.w_sig2 = orc.st["sigma_net.net.2.weight"]

    def __call__(self, x, w):
        lay = self.by_id[id(w)]
        if self.fold and lay == "sig2":
            return torch.cat([self.linear(lay, x, w[:1]), x], dim=-1)
        if self.fold and lay == "col0":
            w_fold = (w[:, 16:144].double() @ self.w_sig2[1:129].double()).float()
            w = torch.cat([w[:, :16], w_fold, w[:, 144:]], dim=1)
        return self.linear(lay, x, w)

    def linear(self, lay, x, w):
        am, wm = self.cfg.get(lay, ("f32", "f32"))
        xs = [x] if am == "f32" else ([r16(x, self.kind)] if am == "x1" else list(split(x, self.kind)))
        ws = [w] if wm == "f32" else ([r16(w, self.kind)] if wm == "x1" else list(split(w, self.kind)))
        out = None
        for i, xa in enumerate(xs):
            for j, wb in enumerate(ws):
                if i == 1 and j == 1:
                    continue      # lo x lo is dropped (as in the x3 scheme)
                t = F.linear(xa, wb)
                out = t if out is None else out + t
        return out


TABLES = ("position_embedder.embeddings", "ambient_embedder.embeddings")


def run(sc, state, fi, cfg, kind, tables16, fold=False, tables=TABLES):
    st = dict(state)
    if tables16:
        for k in tables:
            st[k] = r16(st[k], tables16)
    orc = OracleModel(st, sc.hparams)
    orc.density_scale = sc.density_scale
    emu = Emu(st, kind, cfg, fold)
    emu.bind(orc)
    orc._linear = emu
    return orc.render(fi["rays_o"], fi["rays_d"], fi["cond"], fi["bg_coords"], fi["poses"], bg_color=fi["bg_color"], T_thresh=sc.T_thresh, **sc.hparams)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=64)
    ap.add_argument("--gain", type=float, default=4.0)
    ap.add_argument("--ds", type=float, default=1.0)
    ap.add_argument("--kind", default="fp16")
    ap.add_argument("--fold-only", action="store_true", help="only the kernel modes with and without the sigma-L2 geo fold")
    args = ap.parse_args()
    ops.build()
    sc = scn.Scene(H=args.size, W=args.size, T=4, torso=False, density_scale=args.ds, table_decay=1.0, table_amp=1.0)
    state = lively_state(sc.state, args.gain)
    fi = sc.frame_inputs(0)
    ref = run(sc, state, fi, {}, args.kind, None)

    def report(name, cfg, tables16=None, fold=False, tables=TABLES):
        out = run(sc, state, fi, cfg, args.kind, tables16, fold, tables)
        rep = parity_report(out["rgb_map"].view(-1, 3), ref["rgb_map"].view(-1, 3), ref["knife"], knife_tol=3e-2)
        print(f"{name:58s} max|d|={rep['max_abs']:.2e} (all {rep['max_abs_all']:.2e}, knife {rep['n_knife']}) psnr={rep['psnr']:.1f}", flush=True)

    mma_layers = ["amb0", "amb1", "sig0", "sig1", "sig2", "col0"]     # amb2 / col1 are fp32 dot products in the kernel
    # k_head_v2's two modes with sigma L2's geo rows as separate MMA + fp16 activations ("parent") and folded into color L0
    # (W_fold, "folded").  Robust: the position table is fixed point in the kernel (2^-16 of each level's range), fp32 here.
    kernel_modes = {"fp16 kernel": ({l: ("x1", "x1") for l in mma_layers}, TABLES),
                    "robust kernel": ({**{l: ("x1", "x1") for l in mma_layers}, "amb0": ("x2", "x2"), "amb1": ("x2", "x2")},
                                      ("ambient_embedder.embeddings",))}
    for name, (cfg, tables) in kernel_modes.items():
        for fold in (False, True):
            report(f"{name}, {'folded' if fold else 'parent'} geo (ds {args.ds:g})", cfg, args.kind, fold, tables)
    if args.fold_only:
        return
    report("tables 16-bit only", {}, args.kind)
    report("A x1 all MMA layers", {l: ("x1", "f32") for l in mma_layers})
    report("W x1 all MMA layers", {l: ("f32", "x1") for l in mma_layers})
    report("A x1 + W x1 (the single-pass mode, fp32 tables)", {l: ("x1", "x1") for l in mma_layers})
    report("A x1 + W x1 + tables16 (the fp16 kernel mode)", {l: ("x1", "x1") for l in mma_layers}, args.kind)
    for l in mma_layers:
        report(f"  only {l}: A x1 + W x1", {l: ("x1", "x1")})
    report("A x1 + W x2", {l: ("x1", "x2") for l in mma_layers})
    report("A x2 + W x1", {l: ("x2", "x1") for l in mma_layers})
    report("A x2 + W x2 (x3 scheme)", {l: ("x2", "x2") for l in mma_layers})
    report("A x2 + W x2 + tables16", {l: ("x2", "x2") for l in mma_layers}, args.kind)
    cfg = {l: ("x1", "x1") for l in mma_layers}
    for l in ("amb0", "amb1", "sig0", "sig1", "sig2"):
        cfg[l] = ("x2", "x2")
    report("x3 on amb+sigma nets, x1 on color", cfg)
    report("x3 on amb+sigma nets, x1 on color, tables16", cfg, args.kind)
    cfg2 = {l: ("x1", "x1") for l in mma_layers}
    for l in ("sig0", "sig1", "sig2"):
        cfg2[l] = ("x2", "x2")
    report("x3 on sigma net only", cfg2)
    cfg3 = {l: ("x1", "x1") for l in mma_layers}
    for l in ("amb0", "amb1"):
        cfg3[l] = ("x2", "x2")
    report("x3 on ambient net only", cfg3)


if __name__ == "__main__":
    main()
