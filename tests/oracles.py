"""float64 torch restatements of the texture-image samplers (include/nr_b200.h, NR_TEX_UV and NR_TEX_MIPMAP), shared by the
UV, mip and C-ABI matrix tests.

Both samplers run on the product's own face_index_map / weight_map / depth_map (held bit-exact against the CPU oracle
elsewhere) and are differentiable in the image / pyramid and the light factor, so autograd gives the reference image and
light gradients.  `bg` is a uniform colour (3,) or one colour per item [B,3] (NR_BG_PER_BATCH)."""
import numpy as np
import torch


def _bg(bg, dev):
    bgt = torch.as_tensor(np.asarray(bg, np.float64) if not isinstance(bg, torch.Tensor) else bg, dtype=torch.float64,
                          device=dev)
    return bgt.reshape(-1, 1, 1, 3) if bgt.dim() == 2 else bgt


def oracle_rgb(faces, fim, wmap, dmap, uvs, image, light, bg, fill_back, aa):
    """bilinear UV sampler.  faces [B,F,3,3]; uvs [1|B,F',3,2]; image [1|B,Ht,Wt,3] (differentiable); light [B,F,3] or
    None (differentiable); returns the API rgb [B,3,H,W]."""
    dev = fim.device
    B, F = faces.shape[:2]
    S = fim.shape[-1]
    uvs = uvs.double().expand(B, -1, -1, -1)
    if fill_back:
        uvs = torch.cat((uvs, uvs.flip(2)), dim=1)
    img = image.double().expand(B, -1, -1, -1)
    Ht, Wt = img.shape[1:3]
    cov = fim >= 0
    fi = fim.clamp(min=0).long()                                       # [B,S,S]
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces[..., 2][bidx, fi]                                        # [B,S,S,3] winner's own vertex depths
    w = wmap.permute(0, 2, 3, 1)
    zp = dmap[..., None]
    uvk = uvs[bidx, fi]                                                # [B,S,S,3,2]
    # the pixel's uv and texel positions in fp32 with the sampler's pinned operation order (include/nr_b200.h): one fp32
    # ulp of u moves a tap weight by about 6e-8 x Wt, which would otherwise dominate the per-element comparison of
    # texels that receive only small weights
    lam32 = w.float() * (zp.float() / z.float())
    u32 = uvk.float()
    uv = (lam32[..., 0, None] * u32[..., 0, :] + lam32[..., 1, None] * u32[..., 1, :]) + lam32[..., 2, None] * u32[..., 2, :]
    uv = torch.nan_to_num(uv.clamp(0, 1))
    px, py = (uv[..., 0] * (Wt - 1)).double(), (uv[..., 1] * (Ht - 1)).double()
    ix, iy = px.floor().long().clamp(max=Wt - 1), py.floor().long().clamp(max=Ht - 1)
    wx1, wy1 = px - ix, py - iy
    wx0, wy0 = 1 - wx1, 1 - wy1
    x1, y1 = (ix + 1).clamp(max=Wt - 1), (iy + 1).clamp(max=Ht - 1)
    r0, r1 = Ht - 1 - iy, Ht - 1 - y1

    def tap(r, c):
        t = img[bidx, r, c]                                            # [B,S,S,3]
        if light is not None:
            t = t * light.double()[bidx, fi]
        return t
    rgb = ((wx0 * wy0)[..., None] * tap(r0, ix) + (wx0 * wy1)[..., None] * tap(r1, ix)
           + (wx1 * wy0)[..., None] * tap(r0, x1) + (wx1 * wy1)[..., None] * tap(r1, x1))
    rgb = torch.where(cov[..., None], rgb, _bg(bg, dev)).permute(0, 3, 1, 2)
    if aa:
        rgb = torch.nn.functional.avg_pool2d(rgb, 2, 2)
    return rgb


def mip_levels(H, W):
    """level sizes of the mip pyramid of an H x W image (include/nr_b200.h)"""
    out = [(H, W)]
    while out[-1] != (1, 1):
        h, w = out[-1]
        out.append((max(1, (h + 1) >> 1), max(1, (w + 1) >> 1)))
    return out


def pyramid64(image):
    """float64 (numpy or torch, differentiable) restatement of the build: list of levels [Bt,H_l,W_l,3], row 0 = top."""
    xp = torch if isinstance(image, torch.Tensor) else np
    up = image[:, ::-1] if xp is np else image.flip(1)  # tap coordinates: y up from the bottom row
    out = [up]
    H, W = image.shape[1:3]
    for h, w in mip_levels(H, W)[1:]:
        Hs, Ws = out[-1].shape[1:3]
        x0 = np.arange(w) * 2
        x1 = np.minimum(x0 + 1, Ws - 1)
        y0 = np.arange(h) * 2
        y1 = np.minimum(y0 + 1, Hs - 1)
        if xp is torch:
            x0, x1, y0, y1 = (torch.as_tensor(a, device=image.device) for a in (x0, x1, y0, y1))
        s = out[-1]
        a, b = s[:, y0][:, :, x0], s[:, y0][:, :, x1]
        c, d = s[:, y1][:, :, x0], s[:, y1][:, :, x1]
        out.append(((a + b) + (c + d)) * 0.25)
    return [t[:, ::-1] if xp is np else t.flip(1) for t in out]


def unpack_pyramid(pyr, H, W):
    """packed pyramid [Bt,P,3] -> list of levels [Bt,H_l,W_l,3] (views, so autograd reaches the packed tensor)"""
    out, off = [], 0
    for h, w in mip_levels(H, W):
        out.append(pyr[:, off:off + h * w].reshape(pyr.shape[0], h, w, 3))
        off += h * w
    assert off == pyr.shape[1]
    return out


def lod64(faces, fim, wmap, dmap, uvk, S, Ht, Wt, L):
    """float64 level of detail of every raster pixel from the faces (inverse of the pixel-space vertex matrix)."""
    dev = fim.device
    B = faces.shape[0]
    f64 = faces.double()
    px = 0.5 * (f64[..., 0] * S + S - 1)
    py = 0.5 * (f64[..., 1] * S + S - 1)
    T = torch.stack((px, py, torch.ones_like(px)), dim=-2)           # [B,F,3,3] columns = vertices
    M = torch.linalg.inv_ex(T).inverse                                # rows k: d a_k / dx, d a_k / dy, constant
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand_as(fi)
    Mp = M[bidx, fi]                                                  # [B,S,S,3,3]
    z = f64[..., 2][bidx, fi]                                         # [B,S,S,3]
    w = wmap.double().permute(0, 2, 3, 1)
    zp = dmap.double()[..., None]
    lam = w * (zp / z)
    out = []
    for d in (0, 1):
        q = Mp[..., d] / z
        dl = zp * (q - lam * q.sum(-1, keepdim=True))                 # [B,S,S,3]
        du = (uvk[..., 0] * dl).sum(-1) * (Wt - 1)
        dv = (uvk[..., 1] * dl).sum(-1) * (Ht - 1)
        out.append(du * du + dv * dv)
    lod = 0.5 * torch.log2(torch.maximum(*out))
    return torch.nan_to_num(lod, nan=0.0, neginf=0.0).clamp(0, L - 1)


def lod32(faces, fim, wmap, dmap, uvk, S, Ht, Wt, L):
    """the level of detail as include/nr_b200.h pins it in fp32 (the arguments of lod64; returns float64 holding fp32
    values): the K1 inverse of the pixel-space vertices, d l_k / dx from corner differences, each operation rounded to
    fp32 in the header's order.  Every operation is evaluated in float64 and rounded once more, so a result can differ
    from the product's by an ulp where that double rounding or log2 (log2f is not correctly rounded) lands differently.
    It shows how far the fp32 LOD lies from lod64 -- up to 7e-5 in the C-ABI matrix, from the cancellation in
    qx_k - l_k sx -- and so what of a trilinear comparison comes from the LOD alone."""
    r = lambda t: t.float().double()  # round to fp32
    fma = lambda a, b, c: r(a * b + c)  # a * b of two fp32 values is exact in float64
    B = faces.shape[0]
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=fim.device)[:, None, None].expand_as(fi)
    f = r(faces.detach().double())[bidx, fi]  # [B,S,S,3 corners,3]
    fS = float(S)
    px = [r(r(fma(f[..., k, 0], fS, fS) - 1.0) * 0.5) for k in range(3)]  # to_pixel
    py = [r(r(fma(f[..., k, 1], fS, fS) - 1.0) * 0.5) for k in range(3)]
    n = [r(py[1] - py[2]), r(px[2] - px[1]), r(py[2] - py[0]), r(px[0] - px[2]), r(py[0] - py[1]), r(px[1] - px[0])]
    det = fma(px[1], n[2], fma(px[2], n[4], r(px[0] * n[0])))  # face_inverse
    inv = [r(n[2 * k + d] / det) for k in range(3) for d in (0, 1)]  # inv[3k], inv[3k+1]
    z = [f[..., k, 2] for k in range(3)]
    w = r(wmap.double()).permute(0, 2, 3, 1)
    zp = r(dmap.double())
    lam = [r(w[..., k] * r(zp / z[k])) for k in range(3)]
    out = []
    for d in (0, 1):
        q = [r(inv[2 * k + d] / z[k]) for k in range(3)]
        s = r(r(q[0] + q[1]) + q[2])
        dl = [r(zp * r(q[k] - r(lam[k] * s))) for k in (1, 2)]
        u = [uvk[..., k, 0].double() for k in range(3)]
        v = [uvk[..., k, 1].double() for k in range(3)]
        du = fma(r(u[2] - u[0]), dl[1], r(r(u[1] - u[0]) * dl[0]))
        dv = fma(r(v[2] - v[0]), dl[1], r(r(v[1] - v[0]) * dl[0]))
        a, b = r(float(Wt - 1) * du), r(float(Ht - 1) * dv)
        out.append(r(r(a * a) + r(b * b)))
    lod = r(0.5 * r(torch.log2(torch.fmax(*out))))  # fmaxf: a NaN loses to a number
    return torch.nan_to_num(lod, nan=0.0, neginf=0.0).clamp(0, L - 1)


def oracle_trilinear(faces, fim, wmap, dmap, uvs, image, light, bg, fill_back, aa):
    """float64 trilinear sample on the product's maps; image [1|B,Ht,Wt,3] (differentiable through the float64 pyramid),
    light [B,F,3] or None.  Returns (API rgb [B,3,H,W], raster LOD [B,S,S], L)."""
    Ht, Wt = image.shape[1:3]
    return oracle_trilinear_levels(faces, fim, wmap, dmap, uvs, pyramid64(image.double()), Ht, Wt, light, bg, fill_back, aa)


def oracle_trilinear_levels(faces, fim, wmap, dmap, uvs, levels, Ht, Wt, light, bg, fill_back, aa, lod_fn=None):
    """oracle_trilinear on given pyramid levels [1|B,H_l,W_l,3] (e.g. unpack_pyramid of the packed `textures`); the level
    of detail from `lod_fn` (default lod64)"""
    dev = fim.device
    B = faces.shape[0]
    S = fim.shape[-1]
    uvs = uvs.double().expand(B, -1, -1, -1)
    if fill_back:
        uvs = torch.cat((uvs, uvs.flip(2)), dim=1)
    levels = [l.double().expand(B, -1, -1, -1) for l in levels]
    L = len(levels)
    cov = fim >= 0
    fi = fim.clamp(min=0).long()
    bidx = torch.arange(B, device=dev)[:, None, None].expand(B, S, S)
    z = faces.double()[..., 2][bidx, fi]
    w = wmap.double().permute(0, 2, 3, 1)
    zp = dmap.double()[..., None]
    uvk = uvs[bidx, fi]                                                # [B,S,S,3,2]
    # the pixel's uv and texel positions in fp32 with the sampler's pinned operation order (include/nr_b200.h): at 1024
    # texels one ulp of u is 6e-5 texel, which would otherwise dominate the comparison of the large images
    lam32 = w.float() * (zp.float() / z.float())
    u32 = uvk.float()
    uv = (lam32[..., 0, None] * u32[..., 0, :] + lam32[..., 1, None] * u32[..., 1, :]) + lam32[..., 2, None] * u32[..., 2, :]
    uv = torch.nan_to_num(uv.clamp(0, 1))
    lod = (lod_fn or lod64)(faces, fim, wmap, dmap, uvk, S, Ht, Wt, L)
    lt = light.double()[bidx, fi] if light is not None else None

    def bilinear(img):
        h, wd = img.shape[1:3]
        px, py = (uv[..., 0] * (wd - 1)).double(), (uv[..., 1] * (h - 1)).double()  # fp32 positions, as pinned
        ix, iy = px.floor().long().clamp(max=wd - 1), py.floor().long().clamp(max=h - 1)
        wx1, wy1 = px - ix, py - iy
        wx0, wy0 = 1 - wx1, 1 - wy1
        x1, y1 = (ix + 1).clamp(max=wd - 1), (iy + 1).clamp(max=h - 1)
        r0, r1 = h - 1 - iy, h - 1 - y1

        def tap(r, c):
            t = img[bidx, r, c]
            return t * lt if lt is not None else t
        return ((wx0 * wy0)[..., None] * tap(r0, ix) + (wx0 * wy1)[..., None] * tap(r1, ix)
                + (wx1 * wy0)[..., None] * tap(r0, x1) + (wx1 * wy1)[..., None] * tap(r1, x1))

    samples = torch.stack([bilinear(l) for l in levels], dim=0)      # [L,B,S,S,3]
    l0 = lod.floor()
    f = (lod - l0)[..., None]
    l0 = l0.long()
    l1 = (l0 + 1).clamp(max=L - 1)
    pick = lambda l: samples.gather(0, l[None, ..., None].expand(1, B, S, S, 3))[0]
    rgb = (1 - f) * pick(l0) + f * pick(l1)
    rgb = torch.where(cov[..., None], rgb, _bg(bg, dev)).permute(0, 3, 1, 2)
    if aa:
        rgb = torch.nn.functional.avg_pool2d(rgb, 2, 2)
    return rgb, torch.where(cov, lod, torch.full_like(lod, -1.0)), L
