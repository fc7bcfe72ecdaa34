"""Host-side scene description mirroring the Mitsuba 0.6 plugin/property vocabulary.

Plain-data mirror of what the reference's scene graph holds for the `path` hot path: BSDF plugins
(`diffuse`, `roughconductor`, `roughdielectric`, `coating`; property names as in
src/bsdfs/*.cpp), triangle meshes with an optional `area` emitter child (src/emitters/area.cpp),
a `perspective` sensor (src/sensors/perspective.cpp:126-179), and the integrator / sampler / film /
rfilter properties (src/librender/integrator.cpp:190-225, src/samplers/sobol.cpp:86-102,
src/librender/film.cpp:24-95).  A SceneDesc is what the C-ABI (include/b2mts.h) consumes; the XML
loader (mitsuba_b200/host) produces the same structure from a Mitsuba scene file.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

# named IORs, src/bsdfs/ior.h:39-66
NAMED_IOR = {
    "vacuum": 1.0, "helium": 1.000036, "hydrogen": 1.000132, "air": 1.000277, "carbon dioxide": 1.00045,
    "water": 1.3330, "acetone": 1.36, "ethanol": 1.361, "carbon tetrachloride": 1.461, "glycerol": 1.4729,
    "benzene": 1.501, "silicone oil": 1.52045, "bromine": 1.661, "water ice": 1.31, "fused quartz": 1.458,
    "pyrex": 1.470, "acrylic glass": 1.49, "polypropylene": 1.49, "bk7": 1.5046, "sodium chloride": 1.544,
    "amber": 1.55, "pet": 1.5750, "diamond": 2.419,
}

BSDF_TYPES = {"diffuse": 0, "roughconductor": 1, "roughdielectric": 2, "coating": 3, "null": 4, "twosided": 5, "dielectric": 6,
              "conductor": 7, "plastic": 8}
DISTRIBUTIONS = {"beckmann": 0, "ggx": 1, "phong": 2, "as": 2}


def lookup_ior(value, default: str) -> float:
    """src/bsdfs/ior.h:68-100 lookupIOR: a float wins over a name."""
    if value is None:
        value = default
    if isinstance(value, str):
        return float(NAMED_IOR[value.lower()])
    return float(value)


def _fresnel_dielectric_ext(cos_i, eta):
    """util.cpp:651-681 fresnelDielectricExt in float64 (vectorised), used only for the host-side integral below."""
    cos_i = np.asarray(cos_i, np.float64)
    scale = np.where(cos_i > 0, 1.0 / eta, eta)
    cos_t2 = 1 - (1 - cos_i * cos_i) * scale * scale
    tir = cos_t2 <= 0
    ci = np.abs(cos_i)
    ct = np.sqrt(np.maximum(cos_t2, 0))
    e = np.where(cos_i > 0, eta, 1.0 / eta)
    with np.errstate(invalid="ignore", divide="ignore"):
        rs = (ci - e * ct) / (ci + e * ct)
        rp = (e * ci - ct) / (e * ci + ct)
    return np.where(tir, 1.0, 0.5 * (rs * rs + rp * rp))


def conductor_preset(material: str):
    """RGB (eta, k) of a data/ior material preset as the reference derives it (table mitsuba_b200/data/conductor_presets.txt, generated with
    the reference's own spectrum code by tools/extract_conductor_presets.py)."""
    import os
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "conductor_presets.txt")) as f:
        for line in f:
            t = line.split()
            if t and t[0] == material:
                v = [float.fromhex(x) for x in t[1:7]]
                return tuple(v[:3]), tuple(v[3:])
    raise ValueError(f"unknown conductor material preset {material!r}")


def fresnel_diffuse_reflectance(eta: float) -> float:
    """util.cpp:807-859 fresnelDiffuseReflectance(eta, fast=false): integral of F(sqrt(xi), eta) over xi in [0, 1]
    (composite Simpson in float64 instead of the reference's adaptive Gauss-Lobatto with 1e-5 tolerance)."""
    n = 1 << 14
    xi = np.linspace(0.0, 1.0, n + 1)
    f = _fresnel_dielectric_ext(np.sqrt(xi), eta)
    w = np.ones(n + 1); w[1:-1:2] = 4; w[2:-1:2] = 2
    return float(np.float32((w * f).sum() / (3 * n)))


TEX_FILTERS = {"nearest": 0, "bilinear": 1, "trilinear": 2, "ewa": 3}           # bitmap.cpp:213-230
TEX_WRAP = {"repeat": 0, "clamp": 1, "mirror": 2, "zero": 3, "black": 3, "one": 4, "white": 4}  # bitmap.cpp:324-338


@dataclass
class Texture:
    """`bitmap` texture plugin instance (src/textures/bitmap.cpp, SURVEY.md 8f-4).

    `pixels`: linear float32 image, shape (H, W) (luminance) or (H, W, 3) (RGB), row 0 = top row of the file --
    what Bitmap::convert(.., EFloat, gamma 1) hands to the MIP map (mipmap.h:225-229); file decoding is the loader's job.
    """
    pixels: np.ndarray = None
    filter_type: str = "ewa"
    wrap_u: str = "repeat"
    wrap_v: str = "repeat"
    max_anisotropy: float = 20.0
    uoffset: float = 0.0                   # texture.cpp:82-95
    voffset: float = 0.0
    uscale: float = 1.0
    vscale: float = 1.0

    def average_luminance(self) -> float:
        """Luminance of Texture::getAverage() as a BSDF constructor reads it (bitmap.cpp:501-511 -> mipmap.h getAverage: the float
        running sum of level 0 after clampNegative, in raster order, over the texel count: barray.h:102-124), times the energy-conservation
        scale the BSDF wraps around a texture whose maximum exceeds 1 (bsdf.cpp:88-111)."""
        px = np.maximum(np.ascontiguousarray(self.pixels, np.float32), np.float32(0))
        if px.ndim == 3 and px.shape[2] == 1:
            px = px[:, :, 0]
        n = np.float32(px.shape[0] * px.shape[1])
        mx = float(px.max())
        scale = np.float32(0.99) * (np.float32(1.0) / np.float32(mx)) if mx > 1.0 else np.float32(1.0)
        if px.ndim == 2:
            v = np.cumsum(px.reshape(-1), dtype=np.float32)[-1] / n * scale
            return float(v * np.float32(0.212671) + v * np.float32(0.715160) + v * np.float32(0.072169))   # Spectrum(v).getLuminance()
        avg = [np.cumsum(px[:, :, c].reshape(-1), dtype=np.float32)[-1] / n * scale for c in range(3)]
        return float(avg[0] * np.float32(0.212671) + avg[1] * np.float32(0.715160) + avg[2] * np.float32(0.072169))

    def flat(self) -> dict:
        px = np.ascontiguousarray(self.pixels, np.float32)
        if px.ndim == 3 and px.shape[2] == 1:
            px = px[:, :, 0]
        if px.ndim not in (2, 3) or (px.ndim == 3 and px.shape[2] != 3):
            raise ValueError("The input image has an unsupported pixel format!")  # bitmap.cpp:276-278
        return dict(width=int(px.shape[1]), height=int(px.shape[0]), channels=1 if px.ndim == 2 else 3,
                    filterType=TEX_FILTERS[self.filter_type.lower()], wrapU=TEX_WRAP[self.wrap_u], wrapV=TEX_WRAP[self.wrap_v],
                    maxAnisotropy=float(self.max_anisotropy), uoffset=float(self.uoffset), voffset=float(self.voffset),
                    uscale=float(self.uscale), vscale=float(self.vscale), pixels=np.ascontiguousarray(px))


@dataclass
class Bsdf:
    """One BSDF plugin instance; property names and defaults follow the reference constructors."""
    type: str = "diffuse"
    reflectance: object = (0.5, 0.5, 0.5)                      # diffuse.cpp:75-77; an RGB triple or a Texture (diffuse only)
    specular_reflectance: Sequence[float] = (1.0, 1.0, 1.0)   # roughconductor.cpp:171-172 etc.
    specular_transmittance: Sequence[float] = (1.0, 1.0, 1.0)  # roughdielectric.cpp:186-187
    distribution: str = "beckmann"                             # microfacet.h:99-100
    alpha_u: float = 0.1
    alpha_v: float = 0.1
    sample_visible: bool = True                                # microfacet.h:138
    eta: Sequence[float] = (0.0, 0.0, 0.0)                     # roughconductor eta (RGB), material="none"
    k: Sequence[float] = (1.0, 1.0, 1.0)
    material: str = "none"                                     # conductors: a data/ior preset ("Cu", "Au", ...) overrides eta / k (roughconductor.cpp:174-190)
    ext_eta: object = "air"                                    # roughconductor.cpp:187
    int_ior: object = "bk7"                                    # roughdielectric.cpp:190 / coating.cpp:112
    ext_ior: object = "air"
    thickness: float = 1.0                                     # coating.cpp:126
    sigma_a: Sequence[float] = (0.0, 0.0, 0.0)                 # coating.cpp:129-130
    nested: Optional["Bsdf"] = None                            # coating / twosided child BSDF
    nested_back: Optional["Bsdf"] = None                       # twosided: optional second child (twosided.cpp:89-90)
    diffuse_reflectance: Sequence[float] = (0.5, 0.5, 0.5)     # plastic.cpp:158-159
    nonlinear: bool = False                                    # plastic.cpp:161

    def flat(self) -> dict:
        t = BSDF_TYPES[self.type]
        distr = DISTRIBUTIONS[self.distribution.lower()]
        sv = bool(self.sample_visible) and distr != 2           # microfacet.h:145-148
        # the plugins read the roughness as `m_alphaU->eval(its).average()` of a constant texture (roughconductor.cpp:273-274,
        # roughdielectric.cpp): TSpectrum::average() = (a + a + a) * (1.0f / 3) in float (spectrum.h:481-486), not always a itself
        avg3 = lambda a: float((np.float32(0.0) + np.float32(a) + np.float32(a) + np.float32(a)) * (np.float32(1.0) / np.float32(3)))
        d = dict(type=t, distr=distr, sampleVisible=int(sv), nested=-1,
                 alphaU=avg3(self.alpha_u), alphaV=avg3(self.alpha_v), eta=1.0,
                 thickness=float(self.thickness), reflectance=(0.0, 0.0, 0.0),
                 transmittance=tuple(float(x) for x in self.specular_transmittance),
                 etaC=(0.0, 0.0, 0.0), kC=(1.0, 1.0, 1.0), sigmaA=tuple(float(x) for x in self.sigma_a),
                 nested2=-1, diffuseReflectance=(0.5, 0.5, 0.5) if isinstance(self.diffuse_reflectance, Texture) else tuple(float(x) for x in self.diffuse_reflectance), fdrInt=0.0, fdrExt=0.0,
                 specSamplingWeight=0.0, nonlinear=int(self.nonlinear), texture=-1)
        if t == 0 and isinstance(self.reflectance, Texture):
            d["texture_obj"] = self.reflectance   # resolved to an index by SceneDesc.flat_bsdfs()
            d["reflectance"] = (0.5, 0.5, 0.5)
        elif t == 0:
            d["reflectance"] = tuple(float(x) for x in self.reflectance)
        elif t in (1, 7) and isinstance(self.specular_reflectance, Texture):   # <texture name="specularReflectance" type="bitmap">
            d["texture_obj"] = self.specular_reflectance
            d["reflectance"] = (1.0, 1.0, 1.0)
        else:
            d["reflectance"] = tuple(float(x) for x in self.specular_reflectance)
        if t in (1, 7):  # roughconductor.cpp:187-190, conductor.cpp:172-175
            ext = np.float32(lookup_ior(self.ext_eta, "air"))
            recip = np.float32(1.0) / ext  # Spectrum / Float multiplies by the reciprocal (spectrum.h:415-425)
            eta, k = (self.eta, self.k) if self.material.lower() == "none" else conductor_preset(self.material)
            d["etaC"] = tuple(float(np.float32(x) * recip) for x in eta)  # roughconductor.cpp:189-190
            d["kC"] = tuple(float(np.float32(x) * recip) for x in k)
        if t in (2, 3, 6):
            d["eta"] = float(np.float32(lookup_ior(self.int_ior, "bk7")) / np.float32(lookup_ior(self.ext_ior, "air")))
        if t == 8:  # plastic.cpp:145-161,186-204
            int_ior = self.int_ior if self.int_ior != "bk7" else "polypropylene"
            eta = np.float32(lookup_ior(int_ior, "polypropylene")) / np.float32(lookup_ior(self.ext_ior, "air"))
            d["eta"] = float(eta)
            d["fdrInt"] = fresnel_diffuse_reflectance(1.0 / float(eta))
            d["fdrExt"] = fresnel_diffuse_reflectance(float(eta))
            lum = lambda c: float(c[0]) * 0.212671 + float(c[1]) * 0.715160 + float(c[2]) * 0.072169  # spectrum.h:725-727
            if isinstance(self.diffuse_reflectance, Texture):   # <texture name="diffuseReflectance" type="bitmap">
                d["texture_obj"] = self.diffuse_reflectance
                d["diffuseReflectance"] = (0.5, 0.5, 0.5)
                d_avg = self.diffuse_reflectance.average_luminance()
            else:
                d_avg = lum(self.diffuse_reflectance)
            s_avg = lum(self.specular_reflectance)
            d["specSamplingWeight"] = float(np.float32(s_avg / (d_avg + s_avg)))
        return d


@dataclass
class Medium:
    """A participating medium plugin instance + its phase function (SURVEY.md 8f-1).

    `homogeneous` (src/medium/homogeneous.cpp:156-222): sigma_a / sigma_s RGB, strategy balance|single|manual.
    `heterogeneous` (src/medium/heterogeneous.cpp:182-260, method woodcock): a float32 `gridvolume` density in [0, 1]
    (src/volume/gridvolume.cpp), a constant albedo (`constvolume`), `scale`.  Phase: `isotropic` or `hg` (g).
    """
    type: str = "heterogeneous"
    sigma_a: Sequence[float] = (0.0, 0.0, 0.0)
    sigma_s: Sequence[float] = (0.0, 0.0, 0.0)
    strategy: str = "balance"
    sampling_density: float = 0.0          # strategy manual
    channel: Optional[int] = None          # strategy single
    medium_sampling_weight: float = -1.0
    scale: float = 1.0
    albedo: Sequence[float] = (0.75, 0.75, 0.75)
    density: Optional[np.ndarray] = None   # (nz, ny, nx) float32 in [0, 1]
    aabb_min: Sequence[float] = (0.0, 0.0, 0.0)   # data box of the .vol header (gridvolume.cpp:285-292)
    aabb_max: Sequence[float] = (1.0, 1.0, 1.0)
    to_world: Optional[np.ndarray] = None  # gridvolume `toWorld`
    phase: str = "isotropic"
    g: float = 0.8                         # hg.cpp:49

    def flat(self) -> dict:
        d = dict(type={"homogeneous": 0, "heterogeneous": 1}[self.type], phase={"isotropic": 0, "hg": 1}[self.phase], g=float(self.g),
                 sigmaA=tuple(float(x) for x in self.sigma_a), sigmaS=tuple(float(x) for x in self.sigma_s), strategy=0,
                 samplingDensity=0.0, mediumSamplingWeight=0.0, scale=float(self.scale), albedo=tuple(float(x) for x in self.albedo),
                 res=(0, 0, 0), worldToGrid=(0.0,) * 12, aabbMin=(0.0,) * 3, aabbMax=(0.0,) * 3, density=None)
        if self.type == "homogeneous":
            sa, ss = np.float32(self.sigma_a), np.float32(self.sigma_s)
            st = sa + ss
            w = np.float32(self.medium_sampling_weight)
            if w == -1:  # homogeneous.cpp:168-184
                for i in range(3):
                    if st[i] != 0:
                        alb = ss[i] / st[i]
                        if alb > w:
                            w = alb
                if w > 0:
                    w = max(w, np.float32(0.5))
            d["mediumSamplingWeight"] = float(w)
            strat = self.strategy.lower()
            if strat == "balance":
                d["strategy"] = 0
            elif strat == "single":  # homogeneous.cpp:188-203: the channel with the smallest sigma_t
                d["strategy"] = 1
                ch = int(np.argmin(st)) if self.channel is None else int(self.channel)
                d["samplingDensity"] = float(st[ch])
            elif strat == "manual":
                d["strategy"] = 2
                d["samplingDensity"] = float(self.sampling_density)
            else:
                raise ValueError("Specified an unknown sampling strategy")  # `maximum` is not on the path
        else:
            if self.density is None:
                raise ValueError("No density specified!")  # heterogeneous.cpp:230
            dens = np.ascontiguousarray(self.density, np.float32)
            nz, ny, nx = dens.shape
            lo, hi = np.float64(self.aabb_min), np.float64(self.aabb_max)
            v2w = np.eye(4) if self.to_world is None else np.float64(self.to_world)
            w2v = np.linalg.inv(v2w)
            ext = hi - lo
            S = np.diag([(nx - 1) / ext[0], (ny - 1) / ext[1], (nz - 1) / ext[2], 1.0])
            T = np.eye(4); T[:3, 3] = -lo
            w2g = (S @ T @ w2v).astype(np.float32)  # gridvolume.cpp:186-193
            corners = np.array([[x, y, z, 1.0] for x in (lo[0], hi[0]) for y in (lo[1], hi[1]) for z in (lo[2], hi[2])])
            wc = (corners @ v2w.T)[:, :3].astype(np.float32)
            d.update(res=(nx, ny, nz), worldToGrid=tuple(float(x) for x in w2g[:3].reshape(-1)), aabbMin=tuple(float(x) for x in wc.min(0)),
                     aabbMax=tuple(float(x) for x in wc.max(0)), density=dens)
        return d


@dataclass
class Mesh:
    """A TriMesh after TriMesh::configure (normals already generated or absent = face normals)."""
    P: np.ndarray                       # (nV,3) f32
    idx: np.ndarray                     # (nT,3) u32
    N: Optional[np.ndarray] = None      # (nV,3) f32 or None
    UV: Optional[np.ndarray] = None     # (nV,2) f32 or None
    bsdf: Optional[Bsdf] = None         # None -> shape.cpp:48-72 default
    radiance: Optional[Sequence[float]] = None   # `area` emitter child (area.cpp:64-70)
    sampling_weight: float = 1.0        # emitter.cpp:103
    name: str = ""
    interior: Optional[Medium] = None   # <ref name="interior"> (shape.cpp:160-176); with bsdf None -> `null` BSDF
    exterior: Optional[Medium] = None
    group: int = -1                     # >= 0: member of that `shapegroup` (src/shapes/shapegroup.cpp), vertices in object space


@dataclass
class Instance:
    """<shape type="instance"> (src/shapes/instance.cpp): a shapegroup placed with `toWorld`."""
    group: int
    to_world: np.ndarray                # 4x4 object-to-world (affine)


@dataclass
class EnvMap:
    """<emitter type="envmap"> (src/emitters/envmap.cpp:106-181): a latitude-longitude radiance map around the scene.

    `pixels` is the decoded image as linear float RGB, (H, W, 3), top row first (the reference's Bitmap after convert(..., EFloat));
    `to_world` orients it (default: +Y up, the image centre looks down -Z); `scale` multiplies the radiance."""
    pixels: np.ndarray = None
    scale: float = 1.0
    to_world: Optional[np.ndarray] = None
    sampling_weight: float = 1.0
    to_local: Optional[np.ndarray] = None   # inverse of to_world; derived when absent (tests hand in the reference's own float inverse)

    def matrices(self):
        M64 = np.eye(4) if self.to_world is None else np.asarray(self.to_world, np.float64)
        inv = np.linalg.inv(M64) if self.to_local is None else np.asarray(self.to_local, np.float64)
        return np.ascontiguousarray(M64, np.float32), np.ascontiguousarray(inv, np.float32)


@dataclass
class Camera:
    to_world: np.ndarray                # 4x4 camera-to-world (row major)
    fov: float = 39.3077                # degrees along `fov_axis`
    fov_axis: str = "x"
    near: float = 1e-2                  # sensor.cpp:158
    far: float = 1e4                    # sensor.cpp:160
    width: int = 768                    # film.cpp:30-33
    height: int = 576
    aperture_radius: float = 0.0        # > 0: `thinlens` sensor (src/sensors/thinlens.cpp:132-142)
    focus_distance: float = 0.0         # sensor.cpp:162 (default: farClip)
    crop: tuple | None = None           # (cropOffsetX, cropOffsetY, cropWidth, cropHeight), film.cpp:36-47; None = the whole film

    def film_size(self):
        """(width, height) of the film the integrator sees: the crop window if there is one (Film::getCropSize)."""
        return (self.crop[2], self.crop[3]) if self.crop else (self.width, self.height)

    def xfov(self) -> float:
        """src/librender/sensor.cpp:243-263,293-316."""
        aspect = self.width / self.height
        ax = self.fov_axis.lower()
        if ax == "smaller":
            ax = "y" if aspect > 1 else "x"
        elif ax == "larger":
            ax = "x" if aspect > 1 else "y"
        if ax == "x":
            return self.fov
        if ax == "y":
            return math.degrees(2 * math.atan(math.tan(0.5 * math.radians(self.fov)) * aspect))
        if ax == "diagonal":
            diagonal = 2 * math.tan(0.5 * math.radians(self.fov))
            width = diagonal / math.sqrt(1.0 + 1.0 / (aspect * aspect))
            return math.degrees(2 * math.atan(width * 0.5))
        raise ValueError("fovAxis must be one of smaller, larger, diagonal, x, y")

    def sample_to_camera(self) -> np.ndarray:
        """Inverse of m_cameraToSample, src/sensors/perspective.cpp:133-153 (crop window: relSize / relOffset)."""
        aspect = self.width / self.height
        recip = 1.0 / (self.far - self.near)
        cot = 1.0 / math.tan(math.radians(self.xfov() / 2.0))
        persp = np.array([[cot, 0, 0, 0], [0, cot, 0, 0],
                          [0, 0, self.far * recip, -self.near * self.far * recip], [0, 0, 1, 0]], dtype=np.float64)
        tr = np.eye(4); tr[0, 3] = -1.0; tr[1, 3] = -1.0 / aspect
        sc = np.diag([-0.5, -0.5 * aspect, 1.0, 1.0])
        cam_to_sample = sc @ tr @ persp
        if self.crop:
            ox, oy, cw, ch = self.crop
            ctr = np.eye(4); ctr[0, 3] = -ox / self.width; ctr[1, 3] = -oy / self.height
            csc = np.diag([self.width / cw, self.height / ch, 1.0, 1.0])
            cam_to_sample = csc @ ctr @ cam_to_sample
        return np.linalg.inv(cam_to_sample).astype(np.float32)


@dataclass
class RenderParams:
    """Integrator / sampler / film properties on the path (reference defaults)."""
    spp: int = 4                        # sobol.cpp:88 sampleCount
    sampler: str = "sobol"              # "sobol" | "independent"
    seed: int = 0                       # sobol `scramble`; independent stream seed
    max_depth: int = -1                 # integrator.cpp:199
    rr_depth: int = 5                   # integrator.cpp:193
    strict_normals: bool = False
    hide_emitters: bool = False
    rfilter: str = "gaussian"           # film.cpp:89-95 default
    rfilter_param: float = 0.5          # box: radius; gaussian: stddev
    integrator: str = "path"            # "path" (path.cpp) | "volpath" (volpath.cpp) | "direct" (direct.cpp)
    emitter_samples: int = 1            # direct only: emitterSamples / bsdfSamples (direct.cpp:93-108)
    bsdf_samples: int = 1
    sample_lo: int = 0                  # shard: sample indices [lo,hi) of every pixel
    sample_hi: int = 0                  # 0 -> spp


@dataclass
class SceneDesc:
    meshes: List[Mesh] = field(default_factory=list)
    camera: Optional[Camera] = None
    instances: List["Instance"] = field(default_factory=list)
    env_radiance: Optional[Sequence[float]] = None   # <emitter type="constant"> (src/emitters/constant.cpp:47-52); in Scene::m_emitters it precedes the area emitters (scene.cpp:510-516 vs :322-335)
    env_sampling_weight: float = 1.0
    envmap: Optional["EnvMap"] = None              # <emitter type="envmap">; a scene holds at most one environment emitter (scene.cpp:510-514)

    def flat_bsdfs(self):
        """Flatten the BSDF tree to an array (nested referenced by index); returns (list, per-mesh id)."""
        out, ids, memo = [], [], {}
        self._textures, tmemo = [], {}

        def add(b: Bsdf) -> int:
            if id(b) in memo:
                return memo[id(b)]
            d = b.flat()
            tex = d.pop("texture_obj", None)
            if tex is not None:
                if id(tex) not in tmemo:
                    tmemo[id(tex)] = len(self._textures); self._textures.append(tex)
                d["texture"] = tmemo[id(tex)]
            if b.type == "coating":
                if b.nested is None:
                    raise ValueError("coating: A child BSDF instance is required")  # coating.cpp:157-158
                d["nested"] = add(b.nested)
            if b.type == "twosided":
                if b.nested is None:
                    raise ValueError("A nested one-sided material is required!")  # twosided.cpp:87-88
                d["nested"] = add(b.nested)
                d["nested2"] = d["nested"] if b.nested_back is None else add(b.nested_back)
            out.append(d)
            memo[id(b)] = len(out) - 1
            return memo[id(b)]

        for m in self.meshes:
            b = m.bsdf
            if b is None:  # shape.cpp:48-72
                if m.radiance is None and (m.interior is not None or m.exterior is not None):
                    b = Bsdf("null")
                else:
                    b = Bsdf("diffuse", reflectance=(0.0,) * 3 if m.radiance is not None else (0.5,) * 3)
                m.bsdf = b
            ids.append(add(b))
        return out, ids

    def flat_textures(self):
        """Unique bitmap textures in first-use order (the indices stored in flat_bsdfs()[0][i]["texture"])."""
        self.flat_bsdfs()
        return [t.flat() for t in self._textures]

    def flat_media(self):
        """Unique media in first-use order; returns (list of Medium, per-mesh (interior id, exterior id))."""
        out, memo, ids = [], {}, []

        def add(md):
            if md is None:
                return -1
            if id(md) not in memo:
                memo[id(md)] = len(out); out.append(md)
            return memo[id(md)]

        for m in self.meshes:
            ids.append((add(m.interior), add(m.exterior)))
        return out, ids

    def n_triangles(self) -> int:
        """Unique triangles (instanced geometry counts once)."""
        return int(sum(len(m.idx) for m in self.meshes))

    def n_groups(self) -> int:
        return 1 + max([m.group for m in self.meshes] + [i.group for i in self.instances] + [-1])


def look_at(origin, target, up) -> np.ndarray:
    """src/libcore/transform.cpp:191-214 Transform::lookAt (camera-to-world)."""
    p = np.asarray(origin, np.float64); t = np.asarray(target, np.float64); u = np.asarray(up, np.float64)
    d = t - p; d /= np.linalg.norm(d)
    left = np.cross(u, d); left /= np.linalg.norm(left)
    new_up = np.cross(d, left)
    m = np.eye(4)
    m[:3, 0], m[:3, 1], m[:3, 2], m[:3, 3] = left, new_up, d, p
    return m.astype(np.float32)


# ------------------------------------------------------------------------------------------------
# synthetic scenes (SURVEY.md section 8d).  cbox.xml is not in the reference tree; S1 is authored
# from the classic Cornell measurements.
# ------------------------------------------------------------------------------------------------

def _quad(verts, facing=None):
    """Two triangles (0,1,2),(0,2,3); flip winding so the face normal has positive dot with `facing`."""
    P = np.asarray(verts, np.float32)
    idx = np.array([[0, 1, 2], [0, 2, 3]], np.uint32)
    if facing is not None:
        n = np.cross(P[1] - P[0], P[2] - P[0])
        if np.dot(n, np.asarray(facing, np.float32)) < 0:
            idx = idx[:, ::-1].copy()
    return P, idx


def _merge(parts):
    Ps, Is, off = [], [], 0
    for P, I in parts:
        Ps.append(P); Is.append(I + off); off += len(P)
    return np.concatenate(Ps).astype(np.float32), np.concatenate(Is).astype(np.uint32)


def cornell_box(width=1024, height=1024) -> SceneDesc:
    """S1: 5 walls + short box + tall box + ceiling light = 32 triangles in the 556-unit Cornell cube."""
    white = Bsdf("diffuse", reflectance=(0.73, 0.73, 0.73))
    red = Bsdf("diffuse", reflectance=(0.63, 0.065, 0.05))
    green = Bsdf("diffuse", reflectance=(0.14, 0.45, 0.091))
    light_bsdf = Bsdf("diffuse", reflectance=(0.78, 0.78, 0.78))
    meshes = []
    floor = _quad([(552.8, 0, 0), (0, 0, 0), (0, 0, 559.2), (549.6, 0, 559.2)], (0, 1, 0))
    ceil = _quad([(556, 548.8, 0), (556, 548.8, 559.2), (0, 548.8, 559.2), (0, 548.8, 0)], (0, -1, 0))
    back = _quad([(549.6, 0, 559.2), (0, 0, 559.2), (0, 548.8, 559.2), (556, 548.8, 559.2)], (0, 0, -1))
    P, I = _merge([floor, ceil, back])
    meshes.append(Mesh(P, I, bsdf=white, name="walls"))
    P, I = _quad([(0, 0, 559.2), (0, 0, 0), (0, 548.8, 0), (0, 548.8, 559.2)], (1, 0, 0))
    meshes.append(Mesh(P, I, bsdf=green, name="right"))
    P, I = _quad([(552.8, 0, 0), (549.6, 0, 559.2), (556, 548.8, 559.2), (556, 548.8, 0)], (-1, 0, 0))
    meshes.append(Mesh(P, I, bsdf=red, name="left"))

    def block(top, h):
        top = [np.array(v, np.float32) for v in top]
        c = np.mean(top, axis=0); c[1] = h / 2
        parts = [_quad(top, (0, 1, 0))]
        for i in range(4):
            a, b = top[i], top[(i + 1) % 4]
            q = [(a[0], 0, a[2]), (a[0], h, a[2]), (b[0], h, b[2]), (b[0], 0, b[2])]
            mid = (np.array(q[0]) + np.array(q[2])) / 2
            parts.append(_quad(q, mid - c))
        return _merge(parts)

    P, I = block([(130, 165, 65), (82, 165, 225), (240, 165, 272), (290, 165, 114)], 165)
    meshes.append(Mesh(P, I, bsdf=white, name="short"))
    P, I = block([(423, 330, 247), (265, 330, 296), (314, 330, 456), (472, 330, 406)], 330)
    meshes.append(Mesh(P, I, bsdf=white, name="tall"))
    # light strictly below the ceiling (no coplanar overlap, SURVEY Appendix A tie-breaking)
    P, I = _quad([(343, 548.3, 227), (343, 548.3, 332), (213, 548.3, 332), (213, 548.3, 227)], (0, -1, 0))
    meshes.append(Mesh(P, I, bsdf=light_bsdf, radiance=(17.0, 12.0, 4.0), name="light"))
    cam = Camera(look_at((278, 273, -800), (278, 273, 0), (0, 1, 0)), fov=39.3077, near=10.0, far=2800.0,
                 width=width, height=height)
    return SceneDesc(meshes, cam)


def uv_sphere(center, radius, n_theta=64, n_phi=128, smooth=True, with_uv=False):
    """Latitude/longitude sphere; returns (P, N, UV, idx) with outward winding."""
    c = np.asarray(center, np.float64)
    th = np.linspace(0, math.pi, n_theta + 1)
    ph = np.linspace(0, 2 * math.pi, n_phi + 1)
    T, Ph = np.meshgrid(th, ph, indexing="ij")
    D = np.stack([np.sin(T) * np.cos(Ph), np.cos(T), np.sin(T) * np.sin(Ph)], -1).reshape(-1, 3)
    P = (c + radius * D).astype(np.float32)
    N = D.astype(np.float32) if smooth else None
    UV = np.stack([Ph / (2 * math.pi), T / math.pi], -1).reshape(-1, 2).astype(np.float32) if with_uv else None
    idx = []
    W = n_phi + 1
    for i in range(n_theta):
        for j in range(n_phi):
            a, b, c2, d = i * W + j, i * W + j + 1, (i + 1) * W + j + 1, (i + 1) * W + j
            if i != 0:
                idx.append((a, b, c2))
            if i != n_theta - 1:
                idx.append((a, c2, d))
    idx = np.array(idx, np.uint32)
    # make winding outward
    n = np.cross(P[idx[:, 1]] - P[idx[:, 0]], P[idx[:, 2]] - P[idx[:, 0]])
    cen = P[idx].mean(1) - c.astype(np.float32)
    flip = (n * cen).sum(1) < 0
    idx[flip] = idx[flip][:, ::-1]
    return P, N, UV, idx


def material_ball(bsdf: Bsdf, width=1024, height=1024, n_theta=200, n_phi=200) -> SceneDesc:
    """S2: UV sphere (~80k triangles at 200x200) on a diffuse ground quad under one area light."""
    ground = Bsdf("diffuse", reflectance=(0.5, 0.5, 0.5))
    P, I = _quad([(-8, 0, -8), (-8, 0, 8), (8, 0, 8), (8, 0, -8)], (0, 1, 0))
    meshes = [Mesh(P, I, bsdf=ground, name="ground")]
    P, N, UV, I = uv_sphere((0, 1.0, 0), 1.0, n_theta, n_phi, smooth=True)
    meshes.append(Mesh(P, I, N=N, bsdf=bsdf, name="ball"))
    P, I = _quad([(-1.5, 4.0, -1.5), (-1.5, 4.0, 1.5), (1.5, 4.0, 1.5), (1.5, 4.0, -1.5)], (0, -1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0, 0, 0)), radiance=(20.0, 20.0, 20.0), name="light"))
    P, I = _quad([(-8, 0, 8), (-8, 8, 8), (8, 8, 8), (8, 0, 8)], (0, 0, -1))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0.4, 0.45, 0.6)), name="backdrop"))
    cam = Camera(look_at((0, 2.2, -5.0), (0, 0.9, 0), (0, 1, 0)), fov=35.0, near=0.1, far=100.0,
                 width=width, height=height)
    return SceneDesc(meshes, cam)


def config3_scene(width=1024, height=1024, n_theta=200, n_phi=200) -> SceneDesc:
    """BASELINE.json configs[2]: "material ball roughconductor + roughdielectric (GGX)" -- the S2 set-up with two balls, a GGX rough
    conductor (copper-like eta / k, alpha 0.1) and a GGX rough dielectric (bk7 in air, alpha 0.1), ~160k triangles at 200 x 200."""
    d = material_ball(Bsdf("roughconductor", distribution="ggx", alpha_u=0.1, alpha_v=0.1, eta=(0.2004, 0.9240, 1.1022), k=(3.9129, 2.4528, 2.1421)),
                      width, height, n_theta, n_phi)
    ball = d.meshes[1]
    ball.P = (ball.P + np.array([-1.1, 0, 0], np.float32)).astype(np.float32)
    ball.name = "ball_conductor"
    P, N, UV, I = uv_sphere((1.1, 1.0, 0), 1.0, n_theta, n_phi, smooth=True)
    d.meshes.insert(2, Mesh(P, I, N=N, bsdf=Bsdf("roughdielectric", distribution="ggx", alpha_u=0.1, alpha_v=0.1, int_ior="bk7", ext_ior="air"),
                            name="ball_dielectric"))
    return d


def synthetic_sky(w=1024, h=512, seed=4, sun=400.0) -> np.ndarray:
    """A latitude-longitude radiance map for tests and the bench: blue gradient above the horizon, a small sun (`sun` times brighter
    than the sky, a few texels wide: direct sampling has to find it), a dim ground half, and texel-scale noise (the filtered look-up of
    directly visible background has something to filter).  (h, w, 3) float32, top row first."""
    rng = np.random.default_rng(seed)
    v = (np.arange(h, dtype=np.float64)[:, None] + 0.5) / h           # 0 = zenith, 1 = nadir
    u = (np.arange(w, dtype=np.float64)[None, :] + 0.5) / w
    up = np.clip(1.0 - 2.0 * v, 0.0, 1.0)
    img = np.empty((h, w, 3))
    img[..., 0] = 0.25 + 0.35 * (1 - up) ** 3
    img[..., 1] = 0.40 + 0.35 * (1 - up) ** 3
    img[..., 2] = 0.75 + 0.15 * (1 - up) ** 3
    img[v[:, 0] > 0.5] = (0.12, 0.10, 0.08)
    img *= 0.7 + 0.6 * rng.random((h, w, 1))
    su, sv, r = 0.30, 0.22, 1.5 / h
    d2 = ((np.minimum(np.abs(u - su), 1 - np.abs(u - su)) * 2.0) ** 2 + (v - sv) ** 2) / (r * r)
    img += sun * np.exp(-d2)[..., None] * np.array([1.0, 0.9, 0.7])
    return img.astype(np.float32)


def envmap_scene(width=1024, height=1024, map_width=1024, n_theta=200, n_phi=200) -> SceneDesc:
    """The config-3 material balls without their area light, lit by `synthetic_sky` only (rotated a little so that the sun is not on a
    symmetry axis): the environment is seen directly, by reflection, through the glass ball and by direct sampling."""
    d = config3_scene(width, height, n_theta, n_phi)
    d.meshes = [m for m in d.meshes if m.radiance is None]
    a, b = 0.6, 0.2
    ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    rx = np.array([[1, 0, 0], [0, np.cos(b), -np.sin(b)], [0, np.sin(b), np.cos(b)]])
    M = np.eye(4)
    M[:3, :3] = ry @ rx
    d.envmap = EnvMap(pixels=synthetic_sky(map_width, map_width // 2), scale=1.0, to_world=M.astype(np.float32))
    return d


def checker_image(w=256, h=256, cells=8, seed=5, rgb=True) -> np.ndarray:
    """Procedural test image: coloured checkerboard + fine noise (so that filtering matters), linear float32 in [0, 1]."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w]
    chk = (((x * cells) // w + (y * cells) // h) % 2).astype(np.float32)
    noise = rng.random((h, w)).astype(np.float32)
    lum = np.clip(0.15 + 0.6 * chk + 0.25 * noise, 0.0, 1.0).astype(np.float32)
    if not rgb:
        return lum
    tint = np.stack([0.5 + 0.5 * x / max(w - 1, 1), 0.5 + 0.5 * y / max(h - 1, 1), np.full((h, w), 0.8)], -1).astype(np.float32)
    return (lum[:, :, None] * tint).astype(np.float32)


def textured_scene(width=512, height=512, filter_type="ewa", tex_res=256, wrap="repeat", n_theta=64, n_phi=128, two_sided=False) -> SceneDesc:
    """S2 with bitmap textures (SURVEY.md 8f-4): a ground quad whose uv run 0..4 (wrap mode visible, grazing angles ->
    anisotropic EWA footprints), an RGB-textured sphere, a luminance-textured backdrop, one area light."""
    ground_tex = Texture(checker_image(tex_res, tex_res, 8, 5), filter_type=filter_type, wrap_u=wrap, wrap_v=wrap)
    ball_tex = Texture(checker_image(tex_res, tex_res // 2, 16, 6), filter_type=filter_type, uscale=2.0, voffset=0.25)
    back_tex = Texture(checker_image(tex_res // 2 + 3, tex_res // 4 + 1, 4, 7, rgb=False), filter_type=filter_type, wrap_u="mirror", wrap_v="clamp")
    P, I = _quad([(-8, 0, -8), (-8, 0, 8), (8, 0, 8), (8, 0, -8)], (0, 1, 0))
    UV = np.array([(0, 0), (0, 4), (4, 4), (4, 0)], np.float32)
    gb = Bsdf("diffuse", reflectance=ground_tex)
    meshes = [Mesh(P, I, UV=UV, bsdf=Bsdf("twosided", nested=gb) if two_sided else gb, name="ground")]
    P, N, UV, I = uv_sphere((0, 1.0, 0), 1.0, n_theta, n_phi, smooth=True, with_uv=True)
    meshes.append(Mesh(P, I, N=N, UV=UV, bsdf=Bsdf("diffuse", reflectance=ball_tex), name="ball"))
    P, I = _quad([(-1.5, 4.0, -1.5), (-1.5, 4.0, 1.5), (1.5, 4.0, 1.5), (1.5, 4.0, -1.5)], (0, -1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0, 0, 0)), radiance=(20.0, 20.0, 20.0), name="light"))
    P, I = _quad([(-8, 0, 8), (-8, 8, 8), (8, 8, 8), (8, 0, 8)], (0, 0, -1))
    UV = np.array([(-0.5, 1.5), (-0.5, -0.5), (1.5, -0.5), (1.5, 1.5)], np.float32)[[0, 1, 2, 3]]
    meshes.append(Mesh(P, I, UV=UV, bsdf=Bsdf("diffuse", reflectance=back_tex), name="backdrop"))
    cam = Camera(look_at((0, 2.2, -5.0), (0, 0.9, 0), (0, 1, 0)), fov=35.0, near=0.1, far=100.0, width=width, height=height)
    return SceneDesc(meshes, cam)


def stress_scene(n_instances=100, n_theta=224, n_phi=224, width=2048, height=2048, seed=7, instanced=False) -> SceneDesc:
    """S3: one ~100k-triangle bumpy sphere instanced on a jittered grid (config 5 class): flattened into world-space meshes, or
    (`instanced=True`) one shapegroup + `instance` shapes with scale/translate transforms and one material."""
    rng = np.random.default_rng(seed)
    P0, N0, _, I0 = uv_sphere((0, 0, 0), 1.0, n_theta, n_phi, smooth=True)
    bump = 1.0 + 0.08 * np.sin(9 * P0[:, 0]) * np.sin(7 * P0[:, 1]) * np.sin(11 * P0[:, 2])
    P0 = (P0 * bump[:, None]).astype(np.float32)
    g = int(math.ceil(math.sqrt(n_instances)))
    mats = [Bsdf("diffuse", reflectance=tuple(rng.uniform(0.2, 0.8, 3))) for _ in range(8)]
    meshes, instances = [], []
    if instanced:
        meshes.append(Mesh(P0, I0.copy(), N=N0, bsdf=mats[0], name="proto", group=0))
    for k in range(n_instances):
        gx, gz = k % g, k // g
        s = rng.uniform(0.7, 1.1)
        t = np.array([(gx - g / 2 + 0.5) * 2.6 + rng.uniform(-0.3, 0.3), s * 1.0, (gz - g / 2 + 0.5) * 2.6 + rng.uniform(-0.3, 0.3)])
        if instanced:
            M = np.eye(4); M[:3, :3] *= s; M[:3, 3] = t
            instances.append(Instance(0, M.astype(np.float32)))
        else:
            meshes.append(Mesh((P0 * s + t).astype(np.float32), I0.copy(), N=N0, bsdf=mats[k % 8], name=f"inst{k}"))
    e = g * 1.6 + 2
    P, I = _quad([(-e, 0, -e), (-e, 0, e), (e, 0, e), (e, 0, -e)], (0, 1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0.6, 0.6, 0.6)), name="ground"))
    P, I = _quad([(-e / 2, 9.0, -e / 2), (-e / 2, 9.0, e / 2), (e / 2, 9.0, e / 2), (e / 2, 9.0, -e / 2)], (0, -1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0, 0, 0)), radiance=(6.0, 6.0, 6.0), name="light"))
    cam = Camera(look_at((0, e * 0.9, -e * 1.5), (0, 0.5, 0), (0, 1, 0)), fov=45.0, near=0.1, far=1000.0,
                 width=width, height=height)
    return SceneDesc(meshes, cam, instances=instances)


def cube_mesh(lo, hi):
    """Axis-aligned box with outward-facing triangles (12 triangles, 8 shared vertices)."""
    lo, hi = np.asarray(lo, np.float32), np.asarray(hi, np.float32)
    P = np.array([[x, y, z] for z in (lo[2], hi[2]) for y in (lo[1], hi[1]) for x in (lo[0], hi[0])], np.float32)
    quads = [(0, 2, 3, 1), (4, 5, 7, 6), (0, 1, 5, 4), (2, 6, 7, 3), (0, 4, 6, 2), (1, 3, 7, 5)]
    idx = []
    c = (lo + hi) / 2
    for q in quads:
        for tri in ((q[0], q[1], q[2]), (q[0], q[2], q[3])):
            n = np.cross(P[tri[1]] - P[tri[0]], P[tri[2]] - P[tri[0]])
            if np.dot(n, P[list(tri)].mean(0) - c) < 0:
                tri = tri[::-1]
            idx.append(tri)
    return P, np.array(idx, np.uint32)


def smoke_density(res=128, seed=3) -> np.ndarray:
    """Procedural smoke in [0, 1]: a soft blob modulated by a few sinusoidal octaves ((nz, ny, nx) float32)."""
    rng = np.random.default_rng(seed)
    z, y, x = np.meshgrid(*(np.linspace(0, 1, res, dtype=np.float32),) * 3, indexing="ij")
    r2 = (x - 0.5) ** 2 + (y - 0.45) ** 2 * 0.8 + (z - 0.5) ** 2
    d = np.exp(-r2 / 0.045).astype(np.float32)
    for k in range(1, 5):
        f = rng.uniform(2.0, 5.0, 3) * k
        ph = rng.uniform(0, 2 * math.pi, 3)
        d *= (1.0 + 0.45 / k * np.sin(f[0] * x * 2 * math.pi + ph[0]) * np.sin(f[1] * y * 2 * math.pi + ph[1]) * np.sin(f[2] * z * 2 * math.pi + ph[2])).astype(np.float32)
    d = np.clip(d / d.max(), 0.0, 1.0)
    d[d < 0.02] = 0.0
    return np.ascontiguousarray(d, np.float32)


def smoke_scene(width=512, height=512, res=128, scale=24.0, albedo=(0.9, 0.9, 0.9), phase="isotropic", g=0.0, density=None) -> SceneDesc:
    """S4 (config 4): a res^3 density grid in the unit cube, `heterogeneous` Woodcock medium behind an index-matched
    (BSDF-less) cube, on a diffuse floor under one area light."""
    dens = smoke_density(res) if density is None else density
    med = Medium("heterogeneous", scale=scale, albedo=albedo, density=dens, aabb_min=(0, 0, 0), aabb_max=(1, 1, 1), phase=phase, g=g)
    meshes = []
    P, I = _quad([(-3, 0, -3), (-3, 0, 4), (4, 0, 4), (4, 0, -3)], (0, 1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0.45, 0.45, 0.45)), name="floor"))
    P, I = _quad([(-3, 0, 4), (-3, 5, 4), (4, 5, 4), (4, 0, 4)], (0, 0, -1))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0.3, 0.35, 0.5)), name="backdrop"))
    P, I = cube_mesh((0, 0.001, 0), (1, 1.001, 1))
    meshes.append(Mesh(P, I, bsdf=None, interior=med, name="smoke-bounds"))
    P, I = _quad([(-0.4, 2.6, -0.2), (-0.4, 2.6, 0.9), (0.9, 2.6, 0.9), (0.9, 2.6, -0.2)], (0, -1, 0))
    meshes.append(Mesh(P, I, bsdf=Bsdf("diffuse", reflectance=(0, 0, 0)), radiance=(30.0, 28.0, 24.0), name="light"))
    cam = Camera(look_at((0.5, 1.1, -2.6), (0.5, 0.5, 0.5), (0, 1, 0)), fov=36.0, near=0.05, far=100.0, width=width, height=height)
    sd = SceneDesc(meshes, cam)
    # the grid sits in the cube that bounds it: data box = the cube (offset by the 1 mm lift)
    med.aabb_min, med.aabb_max = (0.0, 0.001, 0.0), (1.0, 1.001, 1.0)
    return sd
