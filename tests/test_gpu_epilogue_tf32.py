"""The torso epilogue's split-tf32 tensor-core MLPs (csrc/torso_kernel.cu, k_epilogue).

  * Accuracy: on the masked pixels of a 512x512 frame of the bench scene and of the torso golden scenes, `deform`, `torso_alpha_map`
    and `torso_rgb_map` are within 1e-5 of a float64 restatement of the torso MLPs on the same inputs (the fp32 frequency and grid
    encodings of the oracle, the grid read where the kernel's own `deform` moved the point).
  * Magnitude robustness: powers of two on the hidden units of both nets, compensated in the next layer, leave the field unchanged
    while its hidden activations span ~1e-4..1e2.  A tf32 hi / lo split keeps fp32's exponent, so the error stays of the same size
    (a 16-bit hi / lo split would lose its low part below ~0.1 there).
  * Mode independence: the torso field does not depend on the head's mlp_precision, and the torso maps do not read the head's
    output, so they are bit-identical in all five modes.
  * No register spills in k_epilogue (CPU only: nvcc cross-compiles)."""
import json
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from genefaceplusplus_b200 import build
from genefaceplusplus_b200 import scene as scn
from helpers import build_model

TOL = 1e-5
GOLDEN_DIR = os.path.join(os.path.dirname(__file__), "golden")
TORSO_GOLDEN = ["torso64_ms16_ds1.npz", "torso48_ms16_ds64.npz"]
PRECISIONS = ["fp32", "fp16", "robust", "bf16x3", "bf16"]


def _render(sc, state, t, precision="fp32"):
    model = build_model(sc, state, precision=precision)
    fi = sc.frame_inputs(t)
    out = model.render(fi["rays_o"].cuda(), fi["rays_d"].cuda(), fi["cond"].cuda(), fi["bg_coords"].cuda(), fi["poses"].cuda(),
                       bg_color=fi["bg_color"].cuda(), T_thresh=sc.T_thresh, **sc.hparams)
    torch.cuda.synchronize()
    mask = model.torso_mask(fi["bg_coords"].cuda()).cpu().view(-1)
    return out, mask, fi


def _mlp64(x, ws):
    for i, w in enumerate(ws):
        x = x @ w.double().t()
        if i != len(ws) - 1:
            x = torch.relu(x)
    return x


def _float64_field(sc, state, fi, mask, deform_out):
    """alpha, colour, deform of the masked pixels: the torso MLPs in float64 on the kernel's inputs."""
    from oracle import ops
    from oracle.render import OracleModel
    orc = OracleModel(state, sc.hparams)
    st = orc.st
    bg = fi["bg_coords"].view(-1, 2)[mask]
    x = bg * orc.torso_shrink
    enc_x = ops.freq_encode(x, 10).double()
    enc_pose = ops.freq_encode(fi["poses"].reshape(-1, 6), 4).double().repeat(x.shape[0], 1)
    parts = [enc_x, enc_pose]
    if sc.hparams["torso_individual_embedding_dim"] > 0:
        parts.append(st["torso_individual_codes"][0].double().repeat(x.shape[0], 1))
    h = torch.cat(parts, dim=-1)
    dx = _mlp64(h, [st[f"torso_deform_net.net.{i}.weight"] for i in range(3)])
    # the canonical lookup where the kernel's deform put the point: the grid's own rounding is not the MLPs' error
    xk = (x + deform_out).clamp(-1, 1).float()
    xf = orc._grid(xk, 1, "torso_embedder.embeddings", "torso_embedder.offsets", orc.per_level_scale_torso).double()
    o = _mlp64(torch.cat([xf, h], dim=-1), [st[f"torso_canonicial_net.net.{i}.weight"] for i in range(3)])
    return torch.sigmoid(o[:, :1]), torch.sigmoid(o[:, 1:]), dx


def _errors(sc, state, t):
    out, mask, fi = _render(sc, state, t)
    assert bool(mask.any())
    deform = out["deform"].cpu()
    alpha64, col64, dx64 = _float64_field(sc, state, fi, mask, deform)
    alpha = out["torso_alpha_map"].cpu().view(-1, 1)[mask]
    bgc = fi["bg_color"].view(-1, 3)[mask].double()
    rgb64 = col64 * alpha64 + bgc * (1 - alpha64)
    rgb = out["torso_rgb_map"].cpu().reshape(-1, 3)[mask]
    return {"deform": (deform.double() - dx64).abs().max().item(), "alpha": (alpha.double() - alpha64).abs().max().item(),
            "rgb": (rgb.double() - rgb64).abs().max().item(), "pixels": int(mask.sum())}


def _scenes():
    out = [("bench512", dict(H=512, W=512, T=8, torso=True, density_scale=8.0))]
    for name in TORSO_GOLDEN:
        m = json.loads(bytes(np.load(os.path.join(GOLDEN_DIR, name))["meta"]).decode())
        out.append((name[:-4], dict(H=m["size"], W=m["size"], T=8, torso=True, max_steps=m["max_steps"], density_scale=m["density_scale"])))
    return out


SCENES = _scenes()


@pytest.mark.gpu
@pytest.mark.parametrize("name,kw", SCENES, ids=[s[0] for s in SCENES])
def test_epilogue_matches_float64(name, kw):
    sc = scn.Scene(**kw)
    for t in (0, 5):
        e = _errors(sc, sc.state, t)
        print(f"[{name}/f{t}] {e['pixels']} torso pixels: max|d| deform {e['deform']:.2e}, alpha {e['alpha']:.2e}, torso rgb {e['rgb']:.2e}")
        assert max(e["deform"], e["alpha"], e["rgb"]) <= TOL, (name, t, e)


def _rescaled(state, lo=-13, hi=7):
    """Hidden unit u of every wide layer times 2^e(u), e cycling over lo..hi, the next layer's column u times 2^-e(u): the same field."""
    out = dict(state)
    for net in ("torso_deform_net", "torso_canonicial_net"):
        w = [state[f"{net}.net.{i}.weight"].clone() for i in range(3)]
        for i in range(2):
            n = w[i].shape[0]
            e = torch.tensor([lo + (u * 7 + 3 * i) % (hi - lo + 1) for u in range(n)], dtype=torch.float32)
            w[i] = w[i] * torch.exp2(e)[:, None]
            w[i + 1] = w[i + 1] * torch.exp2(-e)[None, :]
        for i in range(3):
            out[f"{net}.net.{i}.weight"] = w[i]
    return out


@pytest.mark.gpu
def test_epilogue_error_independent_of_activation_magnitude():
    sc = scn.Scene(H=512, W=512, T=8, torso=True, density_scale=8.0)
    base = _errors(sc, sc.state, 0)
    scaled = _errors(sc, _rescaled(sc.state), 0)
    print(f"[unit scale] {base}")
    print(f"[2^-13..2^7] {scaled}")
    for k in ("deform", "alpha", "rgb"):
        assert scaled[k] <= TOL, (k, scaled)
        assert scaled[k] <= 2 * base[k] + 1e-7, (k, base, scaled)


@pytest.mark.gpu
def test_torso_maps_independent_of_mlp_precision():
    sc = scn.Scene(H=512, W=512, T=8, torso=True, density_scale=8.0)
    ref = None
    for p in PRECISIONS:
        out, _, _ = _render(sc, sc.state, 3, precision=p)
        maps = {k: out[k].cpu() for k in ("torso_alpha_map", "torso_rgb_map", "deform")}
        if ref is None:
            ref = maps
            continue
        for k in maps:
            assert torch.equal(maps[k], ref[k]), (p, k, (maps[k] - ref[k]).abs().max().item())


def test_epilogue_no_spills():
    with tempfile.TemporaryDirectory() as td:
        cmd = [build.NVCC, *build.FLAGS, "-Xptxas=-v", "-c", os.path.join(build.CSRC, "torso_kernel.cu"), "-o", os.path.join(td, "k.o")]
        r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    cur, found = None, None
    for line in r.stderr.splitlines():
        m = re.search(r"Compiling entry function '(\w+)'", line)
        if m:
            cur = m.group(1)
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and cur and re.search(r"\dk_epilogueE", cur):
            found = (int(m.group(1)), int(m.group(2)))
    assert found is not None, r.stderr
    print(f"k_epilogue: {found[0]} bytes spill stores, {found[1]} bytes spill loads")
    assert found == (0, 0)
