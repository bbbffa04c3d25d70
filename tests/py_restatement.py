"""A SECOND, independent restatement of the reference's render loop, in pure Python (TEST INFRASTRUCTURE).

`oracle/rt_oracle.hpp` (C++) is the checker every GPU test compares against; it is pinned by the reference's known-answer
tests only, because the reference itself cannot be built in this image. This module restates the same Rust sources a second
time - recursively, like the reference, straight from a parsed JSON config, sharing no code with the C++ oracle (own Philox,
own vector arithmetic, own camera) - so that `tests/test_oracle_vs_python_restatement.py` can demand bit-identical frames from
two restatements written separately. Python floats are IEEE f64 and never contracted; colour arithmetic goes through
numpy.float32 like the reference's Srgb<f32>.

Citations are file:line under /root/reference/raytracer/src/. The RNG contract (one Philox4x32-10 stream per
(seed, pixel, sample), rand 0.8 float conversions, the reference's draw ORDER) is the repo's, see DESIGN.md §3.
Pure-Python loops: small cases only (a 12x9x2 cover frame takes a few seconds).
"""
import math

import numpy as np

f32 = np.float32
U64 = (1 << 64) - 1


# ---- counter-based RNG: Philox4x32-10 (Salmon et al., SC'11), stream = (seed, pixel, sample) -------------------------
def philox4x32_10(ctr, key):
    c0, c1, c2, c3 = ctr
    k0, k1 = key
    for _ in range(10):
        p0 = 0xD2511F53 * c0
        p1 = 0xCD9E8D57 * c2
        c0, c1, c2, c3 = ((p1 >> 32) ^ c1 ^ k0) & 0xFFFFFFFF, p1 & 0xFFFFFFFF, ((p0 >> 32) ^ c3 ^ k1) & 0xFFFFFFFF, p0 & 0xFFFFFFFF
        k0 = (k0 + 0x9E3779B9) & 0xFFFFFFFF
        k1 = (k1 + 0xBB67AE85) & 0xFFFFFFFF
    return c0, c1, c2, c3


class Stream:
    """u64 draws 2b, 2b+1 come from block b, low word first (rand_core's BlockRng::next_u64)."""

    def __init__(self, seed, pixel, sample):
        self.key = (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
        self.pixel, self.sample, self.block, self.pending = pixel, sample, 0, None

    def next_u64(self):
        if self.pending is not None:
            v, self.pending = self.pending, None
            return v
        w = philox4x32_10((self.block, self.sample, self.pixel, 0), self.key)
        self.block += 1
        self.pending = w[2] | (w[3] << 32)
        return w[0] | (w[1] << 32)

    def gen_f64(self):                      # rand 0.8 Standard: 53 bits * 2^-53
        return (self.next_u64() >> 11) * (1.0 / 9007199254740992.0)

    def gen_range_m1_1(self):               # rand 0.8 UniformFloat::sample_single(-1.0, 1.0)
        bits = (self.next_u64() >> 12) | 0x3FF0000000000000
        value1_2 = np.array([bits], dtype=np.uint64).view(np.float64)[0].item()
        return (value1_2 - 1.0) * 2.0 + -1.0


# ---- Point3D (point3d.rs:52-171) as tuples of Python floats ---------------------------------------------------------
def add(a, b): return (a[0] + b[0], a[1] + b[1], a[2] + b[2])
def sub(a, b): return (a[0] - b[0], a[1] - b[1], a[2] - b[2])
def neg(a): return (-a[0], -a[1], -a[2])
def mul(a, s): return (a[0] * s, a[1] * s, a[2] * s)
def div(a, s): return (a[0] / s, a[1] / s, a[2] / s)
def dot(a, b): return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]
def cross(a, b): return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])
def length_squared(a): return a[0] * a[0] + a[1] * a[1] + a[2] * a[2]


def length(a):                               # distance to the origin, point3d.rs:52-65
    dx, dy, dz = a[0] - 0.0, a[1] - 0.0, a[2] - 0.0
    return math.sqrt(dx * dx + dy * dy + dz * dz)


def unit_vector(a):                          # three divisions, point3d.rs:67-70
    l = length(a)
    return (a[0] / l, a[1] / l, a[2] / l)


def fdiv(a, b):                              # IEEE f64 division: x / 0 is +-inf or NaN, as in Rust, not an exception
    if b == 0.0:
        return math.nan if a == 0.0 or a != a else math.copysign(math.inf, a) * math.copysign(1.0, b)
    return a / b


def fsqrt(x):                                # f64::sqrt: NaN below 0
    return math.sqrt(x) if x >= 0.0 else math.nan


def as_usize(x):                             # Rust `as usize` of a float: saturating, NaN -> 0
    if not x > 0.0:
        return 0
    return U64 if x >= 18446744073709551616.0 else int(x)


def near_zero(a):
    e = 2.220446049250313e-16
    return abs(a[0]) < e and abs(a[1]) < e and abs(a[2]) < e


def random_in_unit_sphere(rng):              # point3d.rs:22-38
    while True:
        p = (rng.gen_range_m1_1(), rng.gen_range_m1_1(), rng.gen_range_m1_1())
        if length_squared(p) < 1.0:
            return p


def vec(d): return (float(d["x"]), float(d["y"]), float(d["z"]))


# ---- Camera (camera.rs:45-84) -----------------------------------------------------------------------------------------
class Camera:
    def __init__(self, c):
        look_from, look_at, vup = vec(c["look_from"]), vec(c["look_at"]), vec(c["vup"])
        theta = float(c["vfov"]) * (math.pi / 180.0)       # f64::to_radians
        half_height = math.tan(theta / 2.0)
        half_width = float(c["aspect"]) * half_height
        w = unit_vector(sub(look_from, look_at))
        u = unit_vector(cross(vup, w))
        v = cross(w, u)
        self.origin = look_from
        self.lower_left_corner = sub(sub(sub(self.origin, mul(u, half_width)), mul(v, half_height)), w)
        self.horizontal = mul(mul(u, 2.0), half_width)
        self.vertical = mul(mul(v, 2.0), half_height)

    def get_ray(self, u, v):
        return self.origin, sub(add(add(self.lower_left_corner, mul(self.horizontal, u)), mul(self.vertical, v)), self.origin)


# ---- the scene ---------------------------------------------------------------------------------------------------------
class World:
    def __init__(self, cfg, textures=None, sky_texture=None, seed=0x5EED, atan2=math.atan2):
        self.cfg, self.seed, self.atan2 = cfg, seed, atan2
        self.width, self.height = int(cfg["width"]), int(cfg["height"])
        self.spp, self.max_depth = int(cfg["samples_per_pixel"]), int(cfg["max_depth"])
        self.camera = Camera(cfg["camera"])
        self.objects = cfg["objects"]
        self.spheres = [(vec(o["center"]), float(o["radius"]), next(iter(o["material"].items()))) for o in self.objects]
        self.lights = [s for s in self.spheres if s[2][0] == "Light"]                     # find_lights, raytracer.rs:220-229
        self.textures = textures or {}        # object index -> uint8 [H, W, 3] (decoded by the caller)
        sky = cfg.get("sky", None)
        self.sky = None if sky is None else ("gradient" if sky.get("texture", "") in ("", None) else sky_texture)
        self.rays = 0

    # Sphere::hit, sphere.rs:46-78 (+ u,v :35-43 for every accepted root)
    def sphere_hit(self, idx, o, d, t_min, t_max):
        center, radius, _ = self.spheres[idx]
        oc = sub(o, center)
        a = length_squared(d)
        half_b = dot(oc, d)
        c = length_squared(oc) - radius * radius
        disc = (half_b * half_b) - (a * c)
        if disc >= 0.0:
            sq = math.sqrt(disc)
            for root in (((-half_b) - sq) / a, ((-half_b) + sq) / a):
                if root < t_max and root > t_min:
                    p = add(o, mul(d, root))
                    normal = div(sub(p, center), radius)
                    front = dot(d, normal) < 0.0
                    n = unit_vector(sub(p, center))
                    u = (self.atan2(n[0], n[2]) / (2.0 * math.pi)) + 0.5
                    v = n[1] * 0.5 + 0.5
                    return {"t": root, "point": p, "normal": normal if front else neg(normal), "front": front, "idx": idx, "u": u, "v": v}
        return None

    def hit_world(self, o, d):               # raytracer.rs:44-59
        self.rays += 1
        closest, rec = 1.7976931348623157e308, None
        for i in range(len(self.spheres)):
            h = self.sphere_hit(i, o, d, 0.001, closest)
            if h is not None:
                closest, rec = h["t"], h
        return rec

    # Material::scatter, materials.rs:44-54 -> None | (ray | None, albedo)
    def scatter(self, o, d, h, rng):
        kind, body = self.spheres[h["idx"]][2]
        if kind == "Light":                                                              # :65-69
            return None, (f32(1.0), f32(1.0), f32(1.0))
        if kind in ("Lambertian", "Texture"):                                            # :84-95, :256-267
            sd = add(h["normal"], random_in_unit_sphere(rng))
            if near_zero(sd):
                sd = h["normal"]
            target = add(h["point"], sd)
            ray = (h["point"], sub(target, h["point"]))
            if kind == "Lambertian":
                return ray, tuple(f32(x) for x in body["albedo"])
            tex = self.textures[h["idx"]]                                                # get_albedo, :236-253
            rot = h["u"] + float(body["h_offset"])
            if rot > 1.0:
                rot = rot - 1.0
            W, H = int(body["width"]), int(body["height"])
            uu, vv = rot * float(W), (1.0 - h["v"]) * float(H - 1)
            base = 3 * (as_usize(math.floor(vv)) * W + as_usize(math.floor(uu)))
            flat = tex.reshape(-1)
            if base + 2 >= flat.size:                                                    # the reference panics (index out of bounds)
                raise IndexError(f"texture index {base + 2} out of bounds for {flat.size} bytes")
            return ray, (f32(flat[base]) / f32(255.0), f32(flat[base + 1]) / f32(255.0), f32(flat[base + 2]) / f32(255.0))
        if kind == "Metal":                                                              # :111-129
            reflected = sub(d, mul(h["normal"], 2.0 * dot(d, h["normal"])))
            nd = add(reflected, mul(random_in_unit_sphere(rng), float(body["fuzz"])))
            if dot(nd, h["normal"]) > 0.0:
                return (h["point"], nd), tuple(f32(x) for x in body["albedo"])
            return "absorbed"
        if kind == "Glass":                                                              # :144-155, :176-199
            ior = float(body["index_of_refraction"])
            ratio = fdiv(1.0, ior) if h["front"] else ior
            ud = unit_vector(d)
            cos_theta = min(dot(neg(ud), h["normal"]), 1.0)
            sin_theta = fsqrt(1.0 - cos_theta * cos_theta)
            reflect_it = ratio * sin_theta > 1.0
            if not reflect_it:
                r0 = fdiv(1.0 - ratio, 1.0 + ratio)
                r0 = r0 * r0
                x = 1.0 - cos_theta
                x2 = x * x
                reflect_it = (r0 + (1.0 - r0) * (x * (x2 * x2))) > rng.gen_f64()          # powi(5) = x * (x^2)^2; drawn only when refraction is possible
            if reflect_it:
                nd = sub(ud, mul(h["normal"], 2.0 * dot(ud, h["normal"])))
            else:
                ct = min(dot(neg(ud), h["normal"]), 1.0)
                perp = mul(add(ud, mul(h["normal"], ct)), ratio)
                par = mul(h["normal"], -1.0 * math.sqrt(abs(1.0 - length_squared(perp))))
                nd = add(perp, par)
            return (h["point"], nd), (f32(1.0), f32(1.0), f32(1.0))
        raise ValueError(kind)

    @staticmethod
    def clamp(v):                             # raytracer.rs:61-69
        return f32(0.0) if v < 0.0 else (f32(1.0) if v > 1.0 else v)

    def ray_color(self, o, d, rng, max_depth, depth):        # raytracer.rs:71-165
        if depth <= 0:
            return f32(0.0), f32(0.0), f32(0.0)
        h = self.hit_world(o, d)
        if h is None:
            ud = unit_vector(d)
            t = self.clamp(f32(0.5) * (f32(ud[1]) + f32(1.0)))
            u = self.clamp(f32(0.5) * (f32(ud[0]) + f32(1.0)))
            if self.sky is None:
                return f32(0.0), f32(0.0), f32(0.0)
            if isinstance(self.sky, str):
                omt = (f32(1.0) - t) * f32(1.0)
                return omt + t * f32(0.5), omt + t * f32(0.7), omt + t * f32(1.0)
            H, W = self.sky.shape[0], self.sky.shape[1]
            x = as_usize(u * f32(W - 1)); y = as_usize((f32(1.0) - t) * f32(H - 1))
            px = self.sky.reshape(-1)[(y * W + x) * 3: (y * W + x) * 3 + 3]
            return tuple(f32(0.7) * f32(px[k]) / f32(255.0) for k in range(3))
        sc = self.scatter(o, d, h, rng)
        if sc == "absorbed":
            return f32(0.0), f32(0.0), f32(0.0)
        ray, albedo = sc
        light = [f32(0.0), f32(0.0), f32(0.0)]
        prob = 0.05 if self.spheres[h["idx"]][2][0] == "Glass" else 0.1
        nl = len(self.lights)
        if nl > 0 and rng.gen_f64() > (1.0 - float(nl) * prob) and depth > ((max_depth - 2) & U64):   # usize wrap of a release build
            for lc, _, _ in self.lights:
                tc = self.ray_color(h["point"], sub(lc, h["point"]), rng, 2, 1)
                for k in range(3):
                    light[k] = light[k] + albedo[k] * tc[k]
            for k in range(3):
                light[k] = light[k] / f32(nl)
        if ray is None:
            return albedo
        tc = self.ray_color(ray[0], ray[1], rng, max_depth, depth - 1)
        return tuple(self.clamp(light[k] + albedo[k] * tc[k]) for k in range(3))

    def render(self):
        """render_line over all rows (raytracer.rs:191-218). Returns (linear mean f32 [h,w,3], rgb8 [h,w,3], rays)."""
        w, h = self.width, self.height
        lin = np.zeros((h, w, 3), np.float32); img = np.zeros((h, w, 3), np.uint8)
        self.rays = 0
        for y in range(h):
            for x in range(w):
                acc = [f32(0.0), f32(0.0), f32(0.0)]
                for s in range(self.spp):
                    rng = Stream(self.seed, y * w + x, s)
                    u = (float(x) + rng.gen_f64()) / (float(w) - 1.0)
                    v = (float(h) - (float(y) + rng.gen_f64())) / (float(h) - 1.0)
                    o, d = self.camera.get_ray(u, v)
                    c = self.ray_color(o, d, rng, self.max_depth, self.max_depth)
                    for k in range(3):
                        acc[k] = acc[k] + c[k]
                scale = f32(1.0) / f32(self.spp)
                for k in range(3):
                    m = scale * acc[k]
                    lin[y, x, k] = m
                    # palette 0.6 Srgb<f32> -> u8: min(x*255, 255) + 2^23, low mantissa bits (round half even)
                    scaled = np.fmin(np.sqrt(m) * f32(255.0), f32(255.0))                # f32::min: a NaN operand is dropped
                    bits = int(np.array([scaled + f32(8388608.0)], np.float32).view(np.uint32)[0])
                    img[y, x, k] = max(bits - 0x4B000000, 0) & 0xFF if bits >= 0x4B000000 else 0
        return lin, img, self.rays
