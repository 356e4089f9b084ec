"""CPU restatement of the reference's cube-map projection transformers (habitat_baselines ProjectionTransformer /
ProjectionConverter forward) on the package's own grids (common/projection.Stitch) or on recorded ones, and a float64
bilinear evaluation with an error bar derived from the float32 rounding, for the projection tests."""
import types

import torch
import torch.nn.functional as F


def stitch_float(stitch, faces, is_depth):
    """[B, n_out, C, h, w] float32 before the dtype conversion: every input sampled at every output pixel
    (grid_sample, align_corners=True, zero padding) on the faces as float32, times the input z-factor for depth,
    summed over the inputs, times the output z-factor for depth."""
    x = torch.stack(faces, dim=1).float()                       # [B, n_in, H, W, C]
    B, n_in = x.shape[:2]
    if is_depth and stitch.in_zfactor is not None:
        x = x * stitch.in_zfactor[:, 0, :, :, None]
    h, w = stitch.out_hw
    outs = []
    for o in range(len(stitch.outputs)):
        per_in = [F.grid_sample(x[:, i].permute(0, 3, 1, 2), stitch.grids[i, o].expand(B, h, w, 2),
                                mode="bilinear", padding_mode="zeros", align_corners=True) for i in range(n_in)]
        out = torch.stack(per_in, dim=1).sum(dim=1)            # [B, C, h, w]
        if is_depth and stitch.out_zfactor is not None:
            out = out * stitch.out_zfactor[o]
        outs.append(out)
    return torch.stack(outs, dim=1)


def stitch(stitch_, faces, is_depth):
    """[B * n_out, h, w, C] in the faces' dtype: what the reference transformer writes to its target key."""
    out = stitch_float(stitch_, faces, is_depth)
    B, n_out, C, h, w = out.shape
    return out.to(faces[0].dtype).permute(0, 1, 3, 4, 2).reshape(B * n_out, h, w, C)


def transform(t, observations):
    """The reference transformer `t`'s forward on CPU tensors: {target: output} for every group of t."""
    return {target: stitch(t.stitch, [observations[u] for u in uuids], is_depth)
            for target, uuids, is_depth in t.groups}


def bilinear64(stitch_, faces, is_depth):
    """[B, n_out, C, h, w] float64: the assigned input of every output pixel (Stitch.face) sampled bilinearly at its
    grid point, all in float64 from the float32 grid and z-factors."""
    x = torch.stack(faces, dim=1).double()                      # [B, n_in, H, W, C]
    B, n_in, H, W, C = x.shape
    if is_depth and stitch_.in_zfactor is not None:
        x = x * stitch_.in_zfactor[:, 0, :, :, None].double()
    outs = []
    for o in range(len(stitch_.outputs)):
        face = stitch_.face[o]
        g = stitch_.grids.permute(1, 0, 2, 3, 4)[o].double()    # [n_in, h, w, 2]
        gi = g.gather(0, face.clamp(min=0)[None, :, :, None].expand(1, *face.shape, 2))[0]
        px = (gi[..., 0] + 1) / 2 * (W - 1)
        py = (gi[..., 1] + 1) / 2 * (H - 1)
        x0, y0 = px.floor(), py.floor()
        fx, fy = px - x0, py - y0
        acc = torch.zeros(B, C, *face.shape, dtype=torch.float64)
        for dy, dx, wt in ((0, 0, (1 - fy) * (1 - fx)), (0, 1, (1 - fy) * fx), (1, 0, fy * (1 - fx)),
                           (1, 1, fy * fx)):
            xi, yi = (x0 + dx).long(), (y0 + dy).long()
            inside = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H) & (face >= 0)
            v = x[:, face.clamp(min=0), yi.clamp(0, H - 1), xi.clamp(0, W - 1)]   # [B, h, w, C]
            acc += (v * (wt * inside).unsqueeze(-1)).permute(0, 3, 1, 2)
        if is_depth and stitch_.out_zfactor is not None:
            acc = acc * stitch_.out_zfactor[o].double()
        outs.append(acc)
    return torch.stack(outs, dim=1)


def error_bar(stitch_, faces, is_depth):
    """Per-output bound on |float32 restatement - float64|.  The sampling point is off by at most 3 roundings of
    x = (g + 1) * (W - 1) / 2 (|dx| <= 3 * 2^-24 * W), which moves the value by at most |dx| times the largest jump
    between neighbouring taps (<= 2 * M, M the largest |input|); the four weights carry 3 roundings each and the
    fma chain 4, each at most 2^-24 * M; the z-factors 2 more.  Doubled for slack."""
    H, W = faces[0].shape[1:3]
    M = max(float(torch.stack(faces).double().abs().max()), 1.0)
    zf = 1.0
    if is_depth and stitch_.in_zfactor is not None:
        zf *= float(stitch_.in_zfactor.max())
    if is_depth and stitch_.out_zfactor is not None:
        zf *= float(stitch_.out_zfactor.max())
    u = 2.0 ** -24
    return 2 * zf * M * u * (3 * max(H, W) * 2 + 12 + 4 + 2)


# the cases of tests/golden/projection.pt: name -> (kind, output (h, w), fisheye (fov, params), face key, face shape
# [B, H, W, C], dtype); the faces are drawn from a CPU generator seeded with the case's position.  Each case records the
# reference's table and depth factors next to its output, because their last bits depend on the host (DESIGN §8.2b).
GOLDEN_CASES = {
    "c2e_rgb": ("c2e", (32, 64), None, "rgb", (2, 16, 16, 3), torch.uint8),
    "c2f_depth": ("c2f", (40, 56), (180, (0.2, 0.2, 0.2)), "depth", (2, 40, 56, 1), torch.float32),
    "c2f_rgb": ("c2f", (40, 56), (180, (0.2, 0.2, 0.2)), "rgb", (2, 12, 12, 3), torch.uint8),
    "c2f_sem": ("c2f", (40, 56), (180, (0.2, 0.2, 0.2)), "semantic", (2, 12, 12, 1), torch.int32),
    "e2c_depth": ("e2c", (24, 24), None, "depth", (2, 256, 512, 1), torch.float32),
}


def golden_faces(name):
    kind, _, _, key, shape, dtype = GOLDEN_CASES[name]
    g = torch.Generator().manual_seed(list(GOLDEN_CASES).index(name))
    out = {}
    for i in range(1 if kind == "e2c" else 6):
        if dtype == torch.uint8:
            out[f"{key}_{i}"] = torch.randint(0, 256, shape, generator=g, dtype=dtype)
        elif dtype == torch.int32:
            out[f"{key}_{i}"] = torch.randint(-2 ** 30, 2 ** 30, shape, generator=g, dtype=dtype)
        else:
            out[f"{key}_{i}"] = torch.rand(shape, generator=g) * 10
    return out


def table_from_grids(grids):
    """[n_out, h, w, 3] (x, y, input) from reference-layout grids [n_in, n_out, h, w, 2]: every pixel's grid point in
    the one input whose grid there is not 2, input -1 where there is none (common/projection.Stitch.table)."""
    g = grids.permute(1, 0, 2, 3, 4)                                  # [n_out, n_in, h, w, 2]
    claimed = (g != 2).all(-1)
    face = torch.where(claimed.any(1), claimed.int().argmax(1), -1)
    pt = g.gather(1, face.clamp(min=0)[:, None, :, :, None].expand(-1, 1, -1, -1, 2))[:, 0]
    pt = torch.where((face >= 0)[..., None], pt, torch.zeros_like(pt))
    return torch.cat([pt, face[..., None].float()], dim=-1).contiguous()


def recorded_stitch(rec):
    """A Stitch-shaped view of a recorded case (table, in_zf, out_zf) for stitch_float / bilinear64: the grids are 2
    wherever the table assigns the pixel to another input."""
    table, n_in = rec["table"], rec["n_in"]
    face = table[..., 2].long()
    grids = torch.stack([torch.where((face == i)[..., None], table[..., :2], torch.full_like(table[..., :2], 2.0))
                         for i in range(n_in)], dim=0)                # [n_in, n_out, h, w, 2]
    zf = lambda t: None if t is None else t[:, None]  # noqa: E731
    return types.SimpleNamespace(grids=grids, face=face, in_zfactor=zf(rec["in_zf"]), out_zfactor=zf(rec["out_zf"]),
                                 out_hw=tuple(table.shape[1:3]), outputs=range(table.shape[0]))


def sqrt_probe_input():
    """Values whose float32 torch.sqrt the recording keeps: the grids' host dependence is torch.sqrt's rounding."""
    return torch.linspace(0.01, 3.0, 4096)
