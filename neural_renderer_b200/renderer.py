"""`Renderer` facade with the reference's attribute bag and three render methods (renderer.py:8-107)."""
from __future__ import annotations

import math

import torch

from . import functional as F
from .rasterize import (DEFAULT_SOFT_GAMMA, DEFAULT_SOFT_SIGMA, rasterize, rasterize_attributes, rasterize_depth,
                        rasterize_silhouettes, rasterize_soft, rasterize_soft_attributes, rasterize_soft_silhouettes)


class Renderer(object):
    def __init__(self):
        # rendering
        self.image_size = 256
        self.anti_aliasing = True
        self.background_color = [0, 0, 0]
        self.fill_back = True

        # camera
        self.perspective = True
        self.viewing_angle = 30
        self.eye = [0, 0, -(1. / math.tan(math.radians(self.viewing_angle)) + 1)]
        self.camera_mode = 'look_at'
        self.camera_direction = [0, 0, 1]
        self.near = 0.1
        self.far = 100

        # light
        self.light_intensity_ambient = 0.5
        self.light_intensity_directional = 0.5
        self.light_color_ambient = [1, 1, 1]  # white
        self.light_color_directional = [1, 1, 1]  # white
        self.light_direction = [0, 1, 0]  # up-to-down
        # specular highlight of shading='phong' (flat and smooth ignore these)
        self.light_intensity_specular = 0.2
        self.light_color_specular = [1, 1, 1]
        self.light_shininess = 64.0
        # extra lights of shading='phong' on top of the light above: a list of F.directional_light / F.point_light
        # records, or one stacked [NL,12] / [1|B,NL,12] tensor (F.light_set), at most 8.  Empty = that light alone
        self.lights = []
        # environment light of shading='phong': irradiance-ready SH coefficients [9,3] / [1|B,9,3]
        # (F.sh_from_environment_map), added to every pixel's diffuse light.  None = no environment
        self.environment_sh = None
        # tangent-space normal map of shading='phong' with a texture image and face_uvs: decoded vectors [Hm,Wm,3] /
        # [1|B,Hm,Wm,3] (F.decode_normal_map), sampled at the same UVs; the tangents come from F.vertex_tangents of the
        # mesh.  It may require grad.  None = the interpolated normals alone
        self.normal_map = None
        # specular map of shading='phong' with a texture image and face_uvs: per texel (ks_r, ks_g, ks_b, shininess)
        # [Hq,Wq,4] / [1|B,Hq,Wq,4] (F.specular_map), sampled at the same UVs; ks multiplies every highlight and the
        # shininess replaces light_shininess.  It may require grad.  None = light_color_specular and light_shininess alone
        self.specular_map = None

        # rasterization
        self.rasterizer_eps = 1e-3

        # not in the reference: fold lighting / fill_back texture handling / vertices_to_faces into the rasterizer (same pixels)
        self.fused = True
        # rasterize.py:389: the reference samples the textures of EVERY batch item with the vertex depths of item 0.
        # None = module default (reference-exact, see neural_renderer_b200.set_reference_exact); False = every item with
        # its own depths (batches of different meshes / cameras, viewpoint shards of a multi-GPU run)
        self.reference_exact = None
        # sampler of a texture image (render(..., face_uvs=...)): 'bilinear', or 'trilinear' through a mip pyramid of the
        # image (minified images neither alias nor leave texels without gradient); per-face cubes ignore it
        self.texture_filter = 'bilinear'
        # 'flat': the reference's one light factor per face; 'smooth': the light evaluated at every vertex from its
        # area-weighted normal and interpolated across the face (Gouraud), with vertex gradients through the normals;
        # 'phong': normal and position interpolated to every pixel, ambient + diffuse + a specular highlight towards `eye`
        # (also with perspective=False: the viewer is a point at `eye`).  Silhouettes and depth ignore it
        self.shading = 'flat'
        # True: render() also sends the vertices the derivative of the colour inside each face (texture moving under the
        # face, smooth light) -- photometric alignment; per-face cubes with a batch > 1 need reference_exact=False
        self.interior_gradient = False

    def _transform(self, vertices):
        # renderer.py:41-50 (look_at / look, then perspective), fused into one kernel on CUDA
        return F.camera_transform(vertices, self.eye, self.camera_mode, self.camera_direction, self.perspective,
                                  self.viewing_angle)

    @staticmethod
    def _fusable(vertices, faces):
        return vertices.is_cuda and faces.is_cuda and vertices.dtype == torch.float32 and not faces.is_floating_point()

    def _indices(self, faces):
        """Face indices as the rasterizer consumes them: a shared (expanded, stride-0) index set stays [1,F,3];
        fill_back appends the reversed copies (renderer.py:38-39) -- index data only, no vertex data is duplicated."""
        if faces.dim() == 3 and faces.shape[0] > 1 and faces.stride(0) == 0:
            faces = faces[:1]
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
        return faces

    def render_silhouettes(self, vertices, faces):
        if self.fused and self._fusable(vertices, faces):
            # vertices_to_faces (renderer.py:51) runs inside the rasterizer: no [B,F,3,3] tensor on either pass
            return rasterize_silhouettes(self._indices(faces), self.image_size, self.anti_aliasing,
                                         vertices=self._transform(vertices))
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
        vertices = self._transform(vertices)
        faces = F.vertices_to_faces(vertices, faces)
        # renderer.py:52 -- near / far / rasterizer_eps are NOT forwarded (module defaults apply)
        return rasterize_silhouettes(faces, self.image_size, self.anti_aliasing)

    def render_soft_silhouettes(self, vertices, faces, sigma=DEFAULT_SOFT_SIGMA):
        """Soft silhouettes [B,H,W] (neural_renderer_b200.rasterize_soft_silhouettes) seen through this renderer's camera,
        with near / far.  Winding does not matter to them, so fill_back adds no copies (a copy would count twice) and the
        result is the same either way; anti_aliasing is ignored (the soft image needs no supersampling).  The gradient
        reaches `vertices` through the camera from every face within reach of a pixel."""
        vertices = self._transform(vertices)
        if self.fused and self._fusable(vertices, faces):
            return rasterize_soft_silhouettes(faces, self.image_size, sigma, self.near, self.far, vertices=vertices)
        return rasterize_soft_silhouettes(F.vertices_to_faces(vertices, faces), self.image_size, sigma, self.near, self.far)

    def render_soft(self, vertices, faces, textures, sigma=DEFAULT_SOFT_SIGMA, gamma=DEFAULT_SOFT_GAMMA, face_uvs=None):
        """Soft RGB images [B,3,H,W] and soft silhouettes [B,H,W] (neural_renderer_b200.rasterize_soft) seen through this
        renderer's camera, with near / far, rasterizer_eps and background_color, lit by the flat light of the faces as
        given (functional.face_light_from_vertices).  textures: per-face cubes [B,F,ts,ts,ts,3] or [1,F,...].  As for the
        soft silhouettes, fill_back adds no copies (a copy would count twice), so a face seen from behind keeps its front
        face's light; anti_aliasing is ignored.  Flat shading only.  The gradient reaches `vertices` through the camera and
        the light, and the textures.  With `face_uvs` [F,3,2] / [B,F,3,2], `textures` is a texture image [Ht,Wt,3] /
        [1|B,Ht,Wt,3] sampled with `self.texture_filter` (as render), and a `face_uvs` with requires_grad gets a
        gradient too."""
        if self.shading != 'flat':
            raise ValueError("render_soft supports shading='flat' only, got shading=%r" % (self.shading,))
        n_lights = self.lights.shape[-2] if isinstance(self.lights, torch.Tensor) else len(self.lights)
        for name, unsupported in (("lights", n_lights), ("environment_sh", self.environment_sh is not None),
                                  ("normal_map", self.normal_map is not None), ("specular_map", self.specular_map is not None)):
            if unsupported:
                raise ValueError("render_soft does not support %s (flat light only)" % name)
        light_args = (self.light_intensity_ambient, self.light_intensity_directional, self.light_color_ambient,
                      self.light_color_directional, self.light_direction)
        args = (self.image_size, sigma, gamma, self.near, self.far, self.rasterizer_eps, self.background_color)
        uv = dict(face_uvs=face_uvs, texture_filter=self.texture_filter if face_uvs is not None else 'bilinear')
        if self.fused and self._fusable(vertices, faces):
            light = F.face_light_from_vertices(vertices, faces, *light_args)
            return rasterize_soft(faces, textures, *args, vertices=self._transform(vertices), face_light=light, **uv)
        light = F.face_light(F.vertices_to_faces(vertices, faces), *light_args)
        return rasterize_soft(F.vertices_to_faces(self._transform(vertices), faces), textures, *args, face_light=light, **uv)

    def render_soft_attributes(self, vertices, faces, vertex_attributes=None, face_attributes=None,
                               sigma=DEFAULT_SOFT_SIGMA, gamma=DEFAULT_SOFT_GAMMA, background=None):
        """Soft attribute images [B,C,H,W] (neural_renderer_b200.rasterize_soft_attributes) seen through this renderer's
        camera, with near / far: e.g. per-vertex colours, `render_soft_attributes(v, f, vertex_attributes=colours)`.
        Exactly one of vertex_attributes [Nv,C] / [1|B,Nv,C] and face_attributes [F,3,C] / [1|B,F,3,C]; background: C
        numbers, a tensor [C] or None (zeros); rasterize_soft_attributes says which can be captured in a CUDA graph.
        As for render_soft, fill_back adds no copies (a copy would count twice) and anti_aliasing is ignored.  No
        lighting.  The gradient reaches `vertices` through the camera from every face within reach of a pixel, and the
        attributes."""
        if (vertex_attributes is None) == (face_attributes is None):
            raise TypeError("give exactly one of vertex_attributes= and face_attributes=")
        args = (self.image_size, sigma, gamma, self.near, self.far)
        transformed = self._transform(vertices)
        if self.fused and self._fusable(vertices, faces):
            return rasterize_soft_attributes(faces, *args, vertices=transformed, vertex_attributes=vertex_attributes,
                                             face_attributes=face_attributes, background=background)
        # op by op: materialised faces, per-vertex attributes gathered to the corners in torch (as render_attributes)
        if vertex_attributes is not None:
            va = vertex_attributes[None] if vertex_attributes.dim() == 2 else vertex_attributes
            B, C = vertices.shape[0], va.shape[-1]
            idx = faces.long().expand(B, -1, -1).reshape(B, -1, 1).expand(-1, -1, C)
            face_attributes = torch.gather(va.expand(B, -1, -1), 1, idx).reshape(B, -1, 3, C)
        return rasterize_soft_attributes(F.vertices_to_faces(transformed, faces), *args, face_attributes=face_attributes,
                                         background=background)

    def render_soft_depth(self, vertices, faces, sigma=DEFAULT_SOFT_SIGMA, gamma=DEFAULT_SOFT_GAMMA):
        """Soft depth maps [B,H,W]: the camera z of the transformed vertices rendered by render_soft_attributes as a
        one-channel per-vertex attribute, with the background at `far` (what render_depth writes where nothing is
        covered).  Every face within reach of a pixel sends its depth a gradient -- hidden faces and faces just outside
        a target outline included -- which the hard depth map does not.

        SoftRas semantics: a pixel within reach of a face but outside it reads (nearly) that face's depth, not `far`.
        The background sits at the normalised depth 1e-3, i.e. just in front of `far`, so its softmax weight is
        exp(-zn / gamma) below that of any reached face at normalised depth zn; even a face's faint edge term D_j
        outweighs it by far at a small gamma.  The soft depth map therefore spreads each silhouette by the cut-off reach
        (about 1.2 px at sigma = 1e-5 and 256 x 256); compare it with a target only where the target is covered, or use
        the soft silhouettes for the outline."""
        transformed = self._transform(vertices)
        args = (self.image_size, sigma, gamma, self.near, self.far)
        # the background made on the device: no host copy, so a step that calls this can be captured in a CUDA graph
        far = torch.full((1,), float(self.far), dtype=torch.float32, device=transformed.device)
        if self.fused and self._fusable(vertices, faces):
            return rasterize_soft_attributes(faces, *args, vertices=transformed, vertex_attributes=transformed[..., 2:3],
                                             background=far)[:, 0]
        fv = F.vertices_to_faces(transformed, faces)
        return rasterize_soft_attributes(fv, *args, face_attributes=fv[..., 2:3], background=far)[:, 0]

    def render_depth(self, vertices, faces):
        if self.fused and self._fusable(vertices, faces):
            return rasterize_depth(self._indices(faces), self.image_size, self.anti_aliasing,
                                   vertices=self._transform(vertices))
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
        vertices = self._transform(vertices)
        faces = F.vertices_to_faces(vertices, faces)
        return rasterize_depth(faces, self.image_size, self.anti_aliasing)  # renderer.py:72

    def render(self, vertices, faces, textures, face_uvs=None):
        """RGB images [B,3,H,W].  `textures` are per-face cubes [B,F,ts,ts,ts,3], or -- with `face_uvs` [F,3,2] /
        [B,F,3,2] (UV of every face corner, OBJ convention) -- a texture image [Ht,Wt,3] / [1|B,Ht,Wt,3] (row 0 = top),
        sampled at the perspective-correct UV with `self.texture_filter` (neural_renderer_b200.rasterize_rgbad).  Both
        the image and a `face_uvs` with requires_grad receive gradients (fused: the fill_back copies' UV gradient is
        folded into the original faces in the kernel; op by op: through the cat / flip of the doubled corners)."""
        texture_filter = self.texture_filter if face_uvs is not None else 'bilinear'
        if self.shading not in ('flat', 'smooth', 'phong'):
            raise ValueError("shading must be 'flat', 'smooth' or 'phong', got %r" % (self.shading,))
        n_lights = self.lights.shape[-2] if isinstance(self.lights, torch.Tensor) else len(self.lights)
        if self.shading != 'phong' and n_lights:
            raise ValueError("lights (a light set) needs shading='phong', got shading=%r" % (self.shading,))
        if self.shading != 'phong' and self.environment_sh is not None:
            raise ValueError("environment_sh (an SH environment) needs shading='phong', got shading=%r" % (self.shading,))
        if self.normal_map is not None:
            if self.shading != 'phong':
                raise ValueError("normal_map needs shading='phong', got shading=%r" % (self.shading,))
            if face_uvs is None:
                raise ValueError("normal_map is addressed by the UVs: it needs a texture image and face_uvs")
        if self.specular_map is not None:
            if self.shading != 'phong':
                raise ValueError("specular_map needs shading='phong', got shading=%r" % (self.shading,))
            if face_uvs is None:
                raise ValueError("specular_map is addressed by the UVs: it needs a texture image and face_uvs")
        fused = (self.fused and self._fusable(vertices, faces) and textures.is_cuda and textures.dtype == torch.float32)
        light_args = (self.light_intensity_ambient, self.light_intensity_directional, self.light_color_ambient,
                      self.light_color_directional, self.light_direction)
        if self.shading == 'smooth':
            return self._render_smooth(vertices, faces, textures, face_uvs, texture_filter, fused, light_args)
        if self.shading == 'phong':
            return self._render_phong(vertices, faces, textures, face_uvs, texture_filter, fused)
        if fused:
            # lighting.py:29-52, renderer.py:78-80 and vertices_to_faces (renderer.py:103) folded into the rasterizer:
            # neither `textures * light`, nor the doubled texture tensor, nor faces [B,F,3,3] exist; pixel values are
            # bit-identical to the op-by-op formulation
            indices = self._indices(faces)
            light = F.face_light_from_vertices(vertices, indices, *light_args)
            return rasterize(
                indices, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                self.background_color, face_light=light, textures_fill_back=self.fill_back,
                vertices=self._transform(vertices), reference_exact=self.reference_exact, face_uvs=face_uvs,
                texture_filter=texture_filter, interior_gradient=self.interior_gradient)
        if face_uvs is not None:
            # op by op: materialised faces, the light factor of those faces (F.face_light), doubled UV corners for fill_back
            if self.fill_back:
                faces = torch.cat((faces, faces.flip(2)), dim=1)
                face_uvs = torch.cat((face_uvs, face_uvs.flip(-2)), dim=-3)
            light = F.face_light(F.vertices_to_faces(vertices, faces), *light_args)
            faces = F.vertices_to_faces(self._transform(vertices), faces)
            return rasterize(
                faces, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                self.background_color, face_light=light, reference_exact=self.reference_exact, face_uvs=face_uvs,
                texture_filter=texture_filter, interior_gradient=self.interior_gradient)
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
            textures = torch.cat((textures, textures.permute(0, 1, 4, 3, 2, 5)), dim=1)
        textures = F.lighting(F.vertices_to_faces(vertices, faces), textures, *light_args)
        vertices = self._transform(vertices)
        faces = F.vertices_to_faces(vertices, faces)
        return rasterize(
            faces, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
            self.background_color, reference_exact=self.reference_exact, interior_gradient=self.interior_gradient)

    def render_attributes(self, vertices, faces, vertex_attributes=None, face_attributes=None):
        """Attribute images [B,C,H,W] (neural_renderer_b200.rasterize_attributes) seen through this renderer's camera:
        e.g. a normal map, `render_attributes(v, f, vertex_attributes=F.vertex_normals(v, f))`.  Exactly one of
        vertex_attributes [Nv,C] / [1|B,Nv,C] and face_attributes [F,3,C] / [1|B,F,3,C] (F = the faces given, without
        fill_back copies: those get the corners reversed).  No lighting, no texture.  Gradients flow into the attributes
        and the vertices (interior derivative; render_silhouettes gives the edge gradient)."""
        if (vertex_attributes is None) == (face_attributes is None):
            raise TypeError("give exactly one of vertex_attributes= and face_attributes=")
        if face_attributes is not None and self.fill_back:
            face_attributes = torch.cat((face_attributes, face_attributes.flip(-2)), dim=-3)
        if self.fused and self._fusable(vertices, faces):
            # per-vertex attributes follow the doubled index set of fill_back as the vertices do
            return rasterize_attributes(self._indices(faces), self.image_size, self.anti_aliasing, self.near, self.far,
                                        self.rasterizer_eps, vertices=self._transform(vertices),
                                        vertex_attributes=vertex_attributes, face_attributes=face_attributes)
        # op by op: materialised faces, per-vertex attributes gathered to the corners in torch
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
        if vertex_attributes is not None:
            va = vertex_attributes[None] if vertex_attributes.dim() == 2 else vertex_attributes
            B, C = vertices.shape[0], va.shape[-1]
            idx = faces.long().expand(B, -1, -1).reshape(B, -1, 1).expand(-1, -1, C)
            face_attributes = torch.gather(va.expand(B, -1, -1), 1, idx).reshape(B, -1, 3, C)
        faces = F.vertices_to_faces(self._transform(vertices), faces)
        return rasterize_attributes(faces, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                                    face_attributes=face_attributes)

    def _render_smooth(self, vertices, faces, textures, face_uvs, texture_filter, fused, light_args):
        # vertex normals of the original faces (the fill_back copies would cancel them), light at every corner of the
        # faces the rasterizer draws (copies: reversed normal), interpolated per pixel and applied to the unlit sample
        if fused:
            indices = self._indices(faces)
            corner = F.corner_light(F.vertex_normals(vertices, faces), indices, *light_args, fill_back=self.fill_back)
            return rasterize(
                indices, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                self.background_color, textures_fill_back=self.fill_back, vertices=self._transform(vertices),
                reference_exact=self.reference_exact, face_uvs=face_uvs, texture_filter=texture_filter,
                corner_light=corner, interior_gradient=self.interior_gradient)
        # op by op: torch normals and light, materialised faces, doubled textures / UV corners for fill_back
        normals = F._vertex_normals_torch(vertices, faces)
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
            if face_uvs is not None:
                face_uvs = torch.cat((face_uvs, face_uvs.flip(-2)), dim=-3)
            else:
                textures = torch.cat((textures, textures.permute(0, 1, 4, 3, 2, 5)), dim=1)
        corner = F._corner_light_torch(normals, faces, *light_args, fill_back=self.fill_back)
        faces = F.vertices_to_faces(self._transform(vertices), faces)
        return rasterize(
            faces, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
            self.background_color, reference_exact=self.reference_exact, face_uvs=face_uvs,
            texture_filter=texture_filter, corner_light=corner, interior_gradient=self.interior_gradient)

    def _light_set(self):
        if isinstance(self.lights, torch.Tensor):
            return self.lights if self.lights.shape[-2] > 0 else None
        return F.light_set(*self.lights) if len(self.lights) else None

    def _render_phong(self, vertices, faces, textures, face_uvs, texture_filter, fused):
        # vertex normals of the original faces, then per corner of the drawn faces (copies: reversed normal) the normal and
        # the world-space position; the light, the specular highlight and the eye (self.eye, world space) are per pixel
        if self.interior_gradient:
            raise ValueError("shading='phong' does not support interior_gradient=True: no vertex gradient flows through the "
                             "per-pixel interpolation of the Phong normal and position")
        params = F.phong_params(self.light_intensity_ambient, self.light_intensity_directional, self.light_intensity_specular,
                                self.light_color_ambient, self.light_color_directional, self.light_color_specular,
                                self.light_direction, self.light_shininess, self.eye, device=vertices.device)
        lights = self._light_set()
        if lights is not None:
            lights = lights.to(vertices.device)
        sh = self.environment_sh
        if sh is not None:
            sh = sh.to(vertices.device)
        nm = self.normal_map
        if nm is not None:
            nm = nm.to(vertices.device)
        sm = self.specular_map
        if sm is not None:
            sm = sm.to(vertices.device)
        if fused:
            indices = self._indices(faces)
            # one mesh seen from B viewpoints (an expanded, stride-0 vertex batch and a shared index set): one corner set
            shared = vertices.shape[0] > 1 and vertices.stride(0) == 0 and indices.shape[0] == 1
            v1, f1 = (vertices[:1], faces[:1]) if shared else (vertices, faces)
            vn = F.vertex_normals(v1, f1)
            cs = F.corner_shading(vn, v1, indices, fill_back=self.fill_back)
            ct = None
            if nm is not None:
                # the shared mesh gets one tangent set too when its UVs are shared ([F,3,2], a batch of 1 or an
                # expanded one); UVs that differ per item give every item the frame of its own UVs
                uv_shared = face_uvs.dim() == 3 or face_uvs.shape[0] == 1 or face_uvs.stride(0) == 0
                if shared and uv_shared:
                    vt = F.vertex_tangents(v1, f1, face_uvs[:1] if face_uvs.dim() == 4 else face_uvs, vn)
                else:
                    vt = F.vertex_tangents(vertices, faces, face_uvs, vn.expand(vertices.shape[0], -1, -1))
                ct = F.corner_tangents(vt, indices, fill_back=self.fill_back)
            return rasterize(
                indices, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
                self.background_color, textures_fill_back=self.fill_back, vertices=self._transform(vertices),
                reference_exact=self.reference_exact, face_uvs=face_uvs, texture_filter=texture_filter,
                corner_shading=cs, shading_params=params, lights=lights, environment_sh=sh, normal_map=nm,
                corner_tangents=ct, specular_map=sm)
        # op by op: torch normals and corners, materialised faces, doubled textures / UV corners for fill_back
        normals = F._vertex_normals_torch(vertices, faces)
        vt = F.vertex_tangents(vertices, faces, face_uvs, normals) if nm is not None else None
        if self.fill_back:
            faces = torch.cat((faces, faces.flip(2)), dim=1)
            if face_uvs is not None:
                face_uvs = torch.cat((face_uvs, face_uvs.flip(-2)), dim=-3)
            else:
                textures = torch.cat((textures, textures.permute(0, 1, 4, 3, 2, 5)), dim=1)
        cs = F._corner_shading_torch(normals, vertices, faces, self.fill_back)
        ct = F.corner_tangents(vt, faces, fill_back=self.fill_back) if vt is not None else None
        faces = F.vertices_to_faces(self._transform(vertices), faces)
        return rasterize(
            faces, textures, self.image_size, self.anti_aliasing, self.near, self.far, self.rasterizer_eps,
            self.background_color, reference_exact=self.reference_exact, face_uvs=face_uvs,
            texture_filter=texture_filter, corner_shading=cs, shading_params=params, lights=lights, environment_sh=sh,
            normal_map=nm, corner_tangents=ct, specular_map=sm)
