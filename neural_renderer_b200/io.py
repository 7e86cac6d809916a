"""OBJ I/O with the reference's conventions (load_obj.py:8-197, save_obj.py:151-191).

File parsing is host-side numpy; the one compute step -- baking a texture image into the per-face ts^3 cubes
(load_obj.py:88-137, a CuPy kernel in the reference) -- runs as `nr_b200_bake_textures` on the GPU, like the
reference needs a GPU for `load_texture=True`.  Results are numpy arrays, as in the reference."""
from __future__ import annotations

import os

import numpy as np


def load_mtl(filename_mtl):
    """Kd colours and map_Kd texture file names per material (load_obj.py:9-22); file order is kept."""
    texture_filenames = {}
    colors = {}
    material_name = ''
    with open(filename_mtl) as f:
        for line in f:
            tok = line.split()
            if not tok:
                continue
            if tok[0] == 'newmtl':
                material_name = tok[1]
            if tok[0] == 'map_Kd':
                texture_filenames[material_name] = tok[1]
            if tok[0] == 'Kd':
                colors[material_name] = np.array([float(v) for v in tok[1:4]], dtype=np.float32)
    return colors, texture_filenames


def _read_image(path):
    """RGB image as float32 in [0, 1] (skimage.io.imread(...) / 255 in the reference, load_obj.py:80)."""
    from PIL import Image
    with Image.open(path) as im:
        return np.asarray(im.convert('RGB'), dtype=np.float32) / np.float32(255.)


def parse_texture_faces(filename_obj):
    """UV triangle per face [F,3,2] and the material name of every face (load_obj.py:27-64)."""
    vt = []
    with open(filename_obj) as f:
        lines = f.readlines()
    for line in lines:
        tok = line.split()
        if tok and tok[0] == 'vt':
            vt.append([float(v) for v in tok[1:3]])
    vt = np.array(vt, dtype=np.float32).reshape(-1, 2)
    faces, material_names, material_name = [], [], ''
    for line in lines:
        tok = line.split()
        if not tok:
            continue
        if tok[0] == 'f':
            vs = tok[1:]
            idx = [int(v.split('/')[1]) if ('/' in v and v.split('/')[1] != '') else 0 for v in vs]
            for i in range(len(vs) - 2):
                faces.append((idx[0], idx[i + 1], idx[i + 2]))
                material_names.append(material_name)
        if tok[0] == 'usemtl':
            material_name = tok[1]
    faces = np.array(faces, dtype=np.int32).reshape(-1, 3) - 1  # a missing index becomes -1 = the last vt, as in the reference
    if vt.shape[0] == 0:
        vt = np.zeros((1, 2), dtype=np.float32)
    uv = vt[faces]                                               # [F,3,2]
    wrap = uv > 1
    uv[wrap] = uv[wrap] % 1                                      # load_obj.py:66
    return np.ascontiguousarray(uv, dtype=np.float32), material_names


def bake_textures(image, uv_faces, is_update, texture_size, textures):
    """The bilinear bake of load_obj.py:88-137 on the GPU (`image` [H,W,3] float32, rows already flipped)."""
    import ctypes

    import torch
    from . import _lib
    if not torch.cuda.is_available():
        raise NotImplementedError("texture baking runs on the GPU (the reference's load_textures needs one as well)")
    lib = _lib.load()
    dev = torch.device("cuda")
    img = torch.from_numpy(np.ascontiguousarray(image, dtype=np.float32)).to(dev)
    uv = torch.from_numpy(np.ascontiguousarray(uv_faces, dtype=np.float32)).to(dev)
    upd = None if is_update is None else torch.from_numpy(np.ascontiguousarray(is_update, dtype=np.int32)).to(dev)
    tex = torch.from_numpy(np.ascontiguousarray(textures, dtype=np.float32)).to(dev)
    with torch.cuda.device(dev):
        stream = ctypes.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        _lib.check(lib.nr_b200_bake_textures(img.data_ptr(), uv.data_ptr(), None if upd is None else upd.data_ptr(),
                                             uv.shape[0], int(texture_size), img.shape[0], img.shape[1], tex.data_ptr(),
                                             stream))
    return tex.cpu().numpy()


def load_textures(filename_obj, filename_mtl, texture_size):
    """Per-face texture cubes [F,ts,ts,ts,3] from the OBJ's UVs and its MTL (load_obj.py:25-144): 0.5 grey, then the
    material's Kd colour, then -- for materials with a map_Kd image -- the bilinear bake."""
    uv_faces, material_names = parse_texture_faces(filename_obj)
    colors, texture_filenames = load_mtl(filename_mtl)
    nf = uv_faces.shape[0]
    textures = np.zeros((nf, texture_size, texture_size, texture_size, 3), dtype=np.float32) + np.float32(0.5)
    names = np.array(material_names)
    for material_name, color in colors.items():
        textures[names == material_name] = color[None, None, None, None, :]
    for material_name, filename_texture in texture_filenames.items():
        path = os.path.join(os.path.dirname(filename_obj), filename_texture)
        image = _read_image(path)[::-1, ::1]                    # load_obj.py:82
        is_update = (names == material_name).astype(np.int32)
        textures = bake_textures(image, uv_faces, is_update, texture_size, textures)
    return textures


def load_texture_image(filename_obj, filename_mtl):
    """The OBJ's materials as ONE texture image plus per-corner UVs, for the rasterizer's texture-image mode:
    (face_uvs [F,3,2] float32, OBJ convention; image [H,W,3] float32, row 0 = top).

    A model whose faces all use one map_Kd image gets that image, unpadded, and its UVs unchanged.  Otherwise every
    map_Kd image used by a face becomes a tile of an atlas with a 1-texel replicated border, faces of materials without
    an image get a 1x1 tile of their Kd colour (0.5 grey without a material, as the cube loader), and the UVs (clamped
    into [0, 1] first) are remapped so that the sample position inside the tile is x0 + u (w - 1), y0 + v (h - 1): a
    bilinear sample of the atlas equals the sample of the material's own image up to the float32 rounding of the UV."""
    uv_faces, material_names = parse_texture_faces(filename_obj)
    colors, texture_filenames = load_mtl(filename_mtl)
    names = np.array(material_names)
    used = list(dict.fromkeys(material_names))  # materials in order of first use
    image_of = {m: texture_filenames[m] for m in used if m in texture_filenames}
    images = {}
    for fn in dict.fromkeys(image_of.values()):
        images[fn] = _read_image(os.path.join(os.path.dirname(filename_obj), fn))
    if len(images) == 1 and len(image_of) == len(used):
        return uv_faces, next(iter(images.values()))
    # tiles: one per image file, one per colour-only material; laid out left to right, top-aligned
    tiles, tile_of = [], {}
    for fn, img in images.items():
        tile_of[fn] = len(tiles)
        tiles.append(img)
    for m in used:
        if m not in image_of:
            color = colors.get(m, np.full(3, 0.5, np.float32))
            tile_of[('color', m)] = len(tiles)
            tiles.append(np.asarray(color, np.float32).reshape(1, 1, 3))
    width = sum(t.shape[1] + 2 for t in tiles)
    height = max(t.shape[0] + 2 for t in tiles)
    atlas = np.zeros((height, width, 3), np.float32)
    placed, x = [], 0
    for t in tiles:
        h, w = t.shape[:2]
        atlas[:h + 2, x:x + w + 2] = np.pad(t, ((1, 1), (1, 1), (0, 0)), mode='edge')
        placed.append((x + 1, h, w))  # first interior column, interior size
        x += w + 2
    uv = np.nan_to_num(np.clip(uv_faces.astype(np.float64), 0.0, 1.0), nan=0.0)
    out = np.empty_like(uv)
    for m in used:
        sel = names == m
        x0, h, w = placed[tile_of[image_of[m]] if m in image_of else tile_of[('color', m)]]
        y0 = height - 1 - h  # tap row (v axis, from the bottom) of the tile's bottom interior row
        out[sel, :, 0] = (x0 + uv[sel, :, 0] * (w - 1)) / (width - 1)
        out[sel, :, 1] = (y0 + uv[sel, :, 1] * (h - 1)) / (height - 1)
    return np.ascontiguousarray(out, dtype=np.float32), atlas


def load_obj(filename_obj, normalization=True, texture_size=4, load_texture=False, texture_mode='cubes'):
    """Load vertices (v x y z), faces (f ...; n-gons are fan-triangulated) and optionally the textures of a Wavefront
    .obj file (load_obj.py:147-197).

    texture_mode='cubes' (the reference's behaviour): returns vertices, faces, textures [F,ts,ts,ts,3] baked from the
    material images.  texture_mode='uv': returns vertices, faces, face_uvs [F,3,2], texture_image [H,W,3] (see
    load_texture_image) for `Renderer.render(vertices, faces, texture_image, face_uvs=face_uvs)`."""
    if texture_mode not in ('cubes', 'uv'):
        raise ValueError("texture_mode must be 'cubes' or 'uv', got %r" % (texture_mode,))
    vertices, faces = [], []
    with open(filename_obj) as f:
        lines = f.readlines()
    for line in lines:
        tok = line.split()
        if not tok:
            continue
        if tok[0] == 'v':
            vertices.append([float(v) for v in tok[1:4]])
        elif tok[0] == 'f':
            vs = [int(t.split('/')[0]) for t in tok[1:]]
            for i in range(len(vs) - 2):
                faces.append((vs[0], vs[i + 1], vs[i + 2]))
    vertices = np.array(vertices, dtype=np.float32)
    faces = np.array(faces, dtype=np.int32) - 1
    textures = None
    if load_texture:
        for line in lines:
            if line.startswith('mtllib'):
                filename_mtl = os.path.join(os.path.dirname(filename_obj), line.split()[1])
                if texture_mode == 'uv':
                    textures = load_texture_image(filename_obj, filename_mtl)
                else:
                    textures = load_textures(filename_obj, filename_mtl, texture_size)
        if textures is None:
            raise Exception('Failed to load textures.')  # load_obj.py:185
    if normalization:  # unit cube centred at zero, load_obj.py:188-192
        vertices -= vertices.min(0)[None, :]
        vertices /= np.abs(vertices).max()
        vertices *= 2
        vertices -= vertices.max(0)[None, :] / 2
    if load_texture and texture_mode == 'uv':
        return (vertices, faces) + textures
    if load_texture:
        return vertices, faces, textures
    return vertices, faces


def create_texture_image(textures, texture_size_out=16):
    """Texture atlas of save_obj.py:10-148: every face gets a texture_size_out^2 tile whose lower-left triangle is the
    face's barycentric texture cube resampled trilinearly; returns (image [H,W,3] float32, rows already flipped for
    writing; uv [F,3,2] in [0,1]).  Vectorised numpy restatement of the reference's two CuPy kernels (the resampling
    pass, then the pass that copies the pixel left of the tile diagonal onto the diagonal's upper neighbour)."""
    textures = np.asarray(textures, dtype=np.float32)
    num_faces, tsi = textures.shape[:2]
    tso = int(texture_size_out)
    tile_width = int((num_faces - 1.) ** 0.5) + 1
    tile_height = int((num_faces - 1.) / tile_width) + 1
    H, W = tile_height * tso, tile_width * tso
    fn_all = np.arange(num_faces)
    column, row = fn_all % tile_width, fn_all // tile_width
    uv = np.zeros((num_faces, 3, 2), np.float32)
    uv[:, 0, 0] = column * tso
    uv[:, 0, 1] = row * tso
    uv[:, 1, 0] = column * tso
    uv[:, 1, 1] = (row + 1) * tso - 1
    uv[:, 2, 0] = (column + 1) * tso - 1
    uv[:, 2, 1] = (row + 1) * tso - 1
    y, x = np.mgrid[0:H, 0:W]
    fn = (x // tso) + (y // tso) * tile_width
    valid = fn < num_faces                      # the reference reads past the arrays for the unused tiles
    fnc = np.where(valid, fn, 0)
    p0, p1, p2 = uv[fnc, 0], uv[fnc, 1], uv[fnc, 2]
    xf, yf = x.astype(np.float32), y.astype(np.float32)
    den = p2[..., 0] * (p0[..., 1] - p1[..., 1]) + p0[..., 0] * (p1[..., 1] - p2[..., 1]) + p1[..., 0] * (p2[..., 1] - p0[..., 1])
    inv = np.stack([
        p1[..., 1] - p2[..., 1], p2[..., 0] - p1[..., 0], p1[..., 0] * p2[..., 1] - p2[..., 0] * p1[..., 1],
        p2[..., 1] - p0[..., 1], p0[..., 0] - p2[..., 0], p2[..., 0] * p0[..., 1] - p0[..., 0] * p2[..., 1],
        p0[..., 1] - p1[..., 1], p1[..., 0] - p0[..., 0], p0[..., 0] * p1[..., 1] - p1[..., 0] * p0[..., 1]], axis=-1) / den[..., None]
    eps = np.float32(1e-5)
    weight = np.stack([inv[..., 3 * k] * xf + inv[..., 3 * k + 1] * yf + inv[..., 3 * k + 2] for k in range(3)], axis=-1)
    weight = weight / (weight.sum(-1, keepdims=True) + eps)
    tif = np.clip(weight * (tsi - 1), 0., tsi - 1 - eps).astype(np.float32)
    ti = tif.astype(np.int32)
    frac = tif - ti
    tex = textures.reshape(num_faces, tsi * tsi * tsi, 3)
    image = np.zeros((H, W, 3), np.float32)
    for pn in range(8):
        wgt = np.ones((H, W), np.float32)
        idx = []
        for k in range(3):
            if (pn >> k) % 2 == 0:
                wgt = wgt * (1 - frac[..., k])
                idx.append(ti[..., k])
            else:
                wgt = wgt * frac[..., k]
                idx.append(np.minimum(ti[..., k] + 1, tsi - 1))  # weight 0 whenever the clamp bites
        isc = idx[0] * tsi * tsi + idx[1] * tsi + idx[2]
        image += wgt[..., None] * tex[fnc, isc]
    image[~valid] = 0
    # second kernel: the pixel just above the tile diagonal takes its left neighbour's colour
    sel = ((y % tso + 1) == (x % tso))
    image[sel] = image[y[sel], x[sel] - 1]
    uv[:, :, 0] /= (W - 1)
    uv[:, :, 1] /= (H - 1)
    return image[::-1], uv


def save_obj(filename, vertices, faces, textures=None):
    """Write a Wavefront .obj (save_obj.py:151-191).  With `textures` [F,ts,ts,ts,3] also the texture atlas
    `<name>.png`, `<name>.mtl` and `vt` / `usemtl` / `f v/vt` lines, so that `load_obj(..., load_texture=True)` reads the
    mesh back."""
    vertices = np.asarray(vertices.detach().cpu() if hasattr(vertices, 'detach') else vertices)
    faces = np.asarray(faces.detach().cpu() if hasattr(faces, 'detach') else faces)
    assert vertices.ndim == 2
    assert faces.ndim == 2
    if textures is not None:
        textures = np.asarray(textures.detach().cpu() if hasattr(textures, 'detach') else textures)
        filename_mtl = filename[:-4] + '.mtl'
        filename_texture = filename[:-4] + '.png'
        material_name = 'material_1'
        texture_image, vertices_textures = create_texture_image(textures)
        from PIL import Image
        # scipy.misc.toimage(image, cmin=0, cmax=1): scale to 0..255, clip, round
        data = (np.clip(texture_image * 255.0, 0, 255) + 0.5).astype(np.uint8)
        Image.fromarray(data, 'RGB').save(filename_texture)
    with open(filename, 'w') as f:
        f.write('# %s\n' % os.path.basename(filename))
        f.write('#\n')
        f.write('\n')
        if textures is not None:
            f.write('mtllib %s\n\n' % os.path.basename(filename_mtl))
        for v in vertices:
            f.write('v %.8f %.8f %.8f\n' % (v[0], v[1], v[2]))
        f.write('\n')
        if textures is not None:
            for v in vertices_textures.reshape((-1, 2)):
                f.write('vt %.8f %.8f\n' % (v[0], v[1]))
            f.write('\n')
            f.write('usemtl %s\n' % material_name)
            for i, face in enumerate(faces):
                f.write('f %d/%d %d/%d %d/%d\n' % (face[0] + 1, 3 * i + 1, face[1] + 1, 3 * i + 2, face[2] + 1, 3 * i + 3))
            f.write('\n')
        else:
            for face in faces:
                f.write('f %d %d %d\n' % (face[0] + 1, face[1] + 1, face[2] + 1))
    if textures is not None:
        with open(filename_mtl, 'w') as f:
            f.write('newmtl %s\n' % material_name)
            f.write('map_Kd %s\n' % os.path.basename(filename_texture))
