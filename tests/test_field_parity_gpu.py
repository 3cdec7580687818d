"""GPU: the fused field kernels (mi3d_field_forward / mi3d_field_backward, csrc/field.cu) element by element against the fp64 restatement
tests/field_ref64.py, called through the C ABI so that each case chooses its row layout: fixed row counts, device counters with the
128-row zero padding, counters above the capacity, two backward chunks, multi-view segment tables.

Every comparison is |got - ref| <= bound with the bound derived per element (field_ref64's docstring states the terms):
  encodings: 16 u of sum |w v| over the 8 corners;  layer GEMMs: 3-term tf32 split forward (3 2^-22 per product, 2 u per add),
  6-term bf16 split backward (2^-21 per product, 2 u per add);  owner arithmetic: a stated multiple of u of the magnitude pass;
  table-gradient entries: the propagated dEnc error plus (contributions + 8) u of (sum |contribution| + |base|), since the REDs and the
  warp-aggregated partial sums add in any order;  weight gradients: the propagated error plus the per-evaluation MMA over 128 rows and
  (evaluations per CTA + 4 CTAs + 64) u of the magnitude for the register / RED sums.
The backward reference starts from the kernel's own tape, which the forward check of the same case holds to the fp64 forward.
Kinks whose fp64 margin lies inside the bound admit both branches; their count is printed and held below 0.1 % of the units / rows.
Output buffers run past the rows the kernels may write and are filled with a NaN pattern no kernel produces; inputs past the sample
count are NaN; gradients accumulate onto a non-zero base.  Each case prints its worst err / bound.
"""
import ctypes as C
import importlib
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import field_ref64 as F
from conftest import load_golden
from helpers import camera_rays, make_table, sphere_bitfield

pytestmark = pytest.mark.gpu

SENT = 0x7FC0BEEF
GUARD = 1000                  # rows past the capacity in every buffer
CHUNK = 65536                 # reference rows per chunk
AMB_MAX = 1e-3                # at most this fraction of kinks may admit both branches
CHUNK_TILES = 8192            # mi3d_field_backward's chunk (field.cu kBwdChunkTiles)


@pytest.fixture(scope="module")
def env():
    L = importlib.import_module("make-it-3d_b200._lib")
    fo = importlib.import_module("make-it-3d_b200.nerf.field_ops")
    lib = L.lib()
    torch.cuda.reset_peak_memory_stats()
    yield SimpleNamespace(L=L, fo=fo, lib=lib, S=torch.cuda.get_device_properties(0).multi_processor_count,
                          ctas=lib.mi3d_field_grid_ctas(C.c_int(0)), scratch=fo.bwd_scratch(torch.device("cuda")), W={}, cases={})
    print(f"\npeak device memory of the field parity tests: {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")


def canvas(n):
    return torch.full((n,), SENT, dtype=torch.int32, device="cuda").view(torch.float32)


def untouched(what, t):
    bad = int((t.view(torch.int32) != SENT).sum())
    assert bad == 0, f"{what}: {bad} elements outside the written rows changed"


class Worst:
    def __init__(self, name):
        self.name, self.r = name, {}

    def add(self, what, got, ref, bound):
        got = got.double()
        exact = bound == 0
        ratio = torch.where(exact, torch.where(got == ref, 0.0, math.inf), (got - ref).abs() / torch.where(exact, 1.0, bound))
        ratio = torch.where(torch.isnan(ratio), math.inf, ratio)
        w = float(ratio.max()) if ratio.numel() else 0.0
        self.r[what] = max(self.r.get(what, 0.0), w)

    def done(self, **counts):
        msg = ", ".join(f"{k} {v:.3g}" for k, v in sorted(self.r.items()))
        extra = ", ".join(f"{k} {v}" for k, v in counts.items())
        print(f"\n[{self.name}] worst err/bound: {msg}" + (f" | {extra}" if extra else ""))
        bad = {k: v for k, v in self.r.items() if not v <= 1.0}
        assert not bad, f"{self.name}: err/bound above 1: {bad}"


# ---------------------------------------------------------------------------------------------------------------------------
# parameters
# ---------------------------------------------------------------------------------------------------------------------------
def weights(env, kind):
    if kind in env.W:
        return env.W[kind]
    log2 = 15 if kind == "hash15" else 19
    hg = env.fo.make_hashgrid(16, 16, float(np.exp2(np.log2(2048 / 16) / 15)), log2)
    n = 2 * hg.n_entries
    if kind == "golden":
        g = load_golden("render_albedo.npz")
        table = make_table(n, int(g["table_seed"]), float(g["table_scale"]))
        ws = [torch.from_numpy(g[k]) for k in ("w1", "b1", "w2", "b2", "w3", "b3")]
    else:                       # table at scale 1, nn.Linear's initialisation: normals are well conditioned
        table = make_table(n, 5, 1.0)
        torch.manual_seed(1)
        lin = [torch.nn.Linear(32, 64), torch.nn.Linear(64, 64), torch.nn.Linear(64, 4)]
        ws = [t.detach() for l in lin for t in (l.weight, l.bias)]
    ws = [t.float().contiguous().cuda() for t in ws]
    table = torch.from_numpy(table).cuda()
    mlp = env.L.Mlp()
    for name, t in zip(("w1", "b1", "w2", "b2", "w3", "b3"), ws):
        setattr(mlp, name, t.data_ptr())
    f64 = F.Field64(F.Grid.from_struct(hg, table), F.Mlp(*ws), 1.0, 5.0, 0.1)
    env.W[kind] = SimpleNamespace(hg=hg, table=table, ws=ws, mlp=mlp, f64=f64, n_entries=hg.n_entries)
    return env.W[kind]


# ---------------------------------------------------------------------------------------------------------------------------
# row layouts
# ---------------------------------------------------------------------------------------------------------------------------
def march(env, HW, radius, seed=3):
    ro, rd, _ = camera_rays(HW)
    N = HW * HW
    cap = N * 64
    dev = "cuda"
    xyzs, dirs = torch.zeros(cap, 3, device=dev), torch.zeros(cap, 3, device=dev)
    deltas, rays = torch.zeros(cap, 2, device=dev), torch.zeros(N, 3, dtype=torch.int32, device=dev)
    counter = torch.zeros(2, dtype=torch.int32, device=dev)
    nears, fars = torch.zeros(N, device=dev), torch.zeros(N, device=dev)
    aabb = torch.tensor([-1, -1, -1, 1, 1, 1], dtype=torch.float32, device=dev)
    noises = torch.from_numpy(np.random.default_rng(seed).random(N, dtype=np.float32)).cuda()
    bits = torch.from_numpy(sphere_bitfield(radius)).cuda()
    scan = torch.empty(env.lib.mi3d_march_rays_train_workspace_bytes(C.c_uint32(N)), dtype=torch.uint8, device=dev)
    ro_, rd_ = torch.from_numpy(ro).cuda(), torch.from_numpy(rd).cuda()
    p = env.L.ptr
    env.L.check(env.lib.mi3d_march_rays_train(p(ro_), p(rd_), p(bits), C.c_float(1.0), C.c_float(0.0), C.c_uint32(512), C.c_uint32(N),
                                              C.c_uint32(1), C.c_uint32(128), C.c_uint32(cap), C.c_void_p(0), C.c_void_p(0), p(aabb),
                                              C.c_float(0.2), p(nears), p(fars), p(noises), C.c_uint64(0), p(xyzs), p(dirs), p(deltas),
                                              p(rays), p(counter), p(scan), env.L.stream()), "march_rays_train")
    M = int(counter[0])
    return xyzs[:M].clone(), dirs[:M].clone()


def integer_u_points(n, levels):
    """points whose fp32 fmaf(scale, u, 0.5f) is an integer for one of `levels` (bound 1: p = 2u - 1 and back are exact)"""
    out = []
    rng = np.random.default_rng(9)
    one, two = np.float32(1), np.float32(2)
    for i in range(n):
        s = float(np.float32(levels[i % len(levels)]))
        pt = []
        for _ in range(3):
            found = None
            for k in rng.permutation(np.arange(int(s) // 2 + 1, int(s))):       # u in (0.5, 1): s u + 0.5 steps by s 2^-24 per ulp
                u0 = np.float32((k - 0.5) / s)
                for step in range(8):
                    u = u0
                    for _ in range(step // 2):
                        u = np.nextafter(u, two if step % 2 else -two, dtype=np.float32)
                    pos = np.float32(float(u) * s + 0.5)
                    if pos == np.floor(pos) and np.float32((np.float32(two * u - one) + one) / two) == u:
                        found = u
                        break
                if found is not None:
                    break
            assert found is not None, "no fp32 u with an integer cell coordinate"
            u = found
            pt.append(np.float32(two * u - one))
        out.append(pt)
    return np.array(out, np.float32)


def splice_adversarial(x, d, W):
    """runs of 32 and 33 identical positions across a warp and a tile boundary, points on the +-bound faces and at u = 1, and points
    whose u * scale + 0.5 is an integer"""
    x, d = x.clone(), d.clone()
    x[16:48] = x[16]; d[16:48] = d[16]
    x[112:145] = x[112]; d[112:145] = d[112]
    faces = torch.tensor([[1, 1, 1], [-1, -1, -1], [1, 0.1, -0.2], [-1, 0.3, 0.05], [0.2, 1, 0.1], [0.1, -1, 1], [0.05, 0.1, 1],
                          [-0.2, 0.3, -1], [0.999, 0.999, 0.1], [1, 1, -1], [-1, 1, 1], [0.0, 0.0, 1.0]], dtype=torch.float32)
    x[200:212] = faces.cuda()
    ints = integer_u_points(16, [W.hg.scales[l] for l in (2, 5, 9, 12)])
    x[212:228] = torch.from_numpy(ints).cuda()
    return x, d


def layout(env, name):
    """cached row layouts: dict(x, d, M, cap, counter/m_fixed/align, segs, nv, mpad[], light[nv,3], smooth_noise)"""
    if name in env.cases:
        return env.cases[name]
    W = weights(env, "unit")
    S = env.S
    l0 = torch.tensor([0.3, 0.5, 0.81]); l0 = l0 / l0.norm()
    cs = SimpleNamespace(segs=None, nv=1, counter=None, m_fixed=0, align=0, noise_mode=0, seed=1234567, views=None)
    if name == "fixed":                     # m_fixed ray-ordered samples, align 0: at most one tile per CTA, the last one partial
        M = (S - 3) * 128 + 77
        x, d = march(env, 40, 0.25)
        assert x.shape[0] >= M
        x, d = splice_adversarial(x[:M], d[:M], W)
        cs.m_fixed, cs.cap, cs.m_pad = M, M + 300, M
    elif name in ("march", "over_cap", "multiview"):
        x, d = march(env, 40, 0.25)
        x, d = splice_adversarial(x, d, W)
        M = x.shape[0]
        cs.counter = torch.tensor([M, 0], dtype=torch.int32, device="cuda")
        cs.align = 128
        if name == "over_cap":              # counter[0] > cap, cap not a multiple of 128: the kernels see min(counter, cap) samples
            cs.cap = (M - 1000) // 128 * 128 + 57
            cs.m_pad = M = cs.cap
        else:
            cs.cap, cs.m_pad = M + 128 + 300, M + 128 - M % 128
        if name == "multiview":             # 3 views, uneven counts; view 2's zero rows belong to another rank
            cuts = [0, M // 5, M // 5 + M // 2, M]
            cnt = [cuts[i + 1] - cuts[i] for i in range(3)]
            pads = [128 - c % 128 for c in cnt]
            bounds = cuts + [M + pads[0], M + pads[0] + pads[1], M + pads[0] + pads[1]]
            segs = env.L.ViewSegs()
            segs.n_views = 3
            for i, b in enumerate(bounds):
                segs.bounds[i] = b
            mpad = [cnt[0] + pads[0], cnt[1] + pads[1], cnt[2] + pads[2] + 5000]
            for i, v in enumerate(mpad):
                segs.mpad[i] = v
            raw = np.frombuffer(bytes(segs), dtype=np.int32).copy()
            cs.segs, cs.segs_host, cs.nv, cs.mpad = torch.from_numpy(raw).cuda(), segs, 3, mpad
            cs.m_pad = bounds[-1]
            cs.counter = None
            lights = torch.nn.functional.normalize(torch.tensor([[0.3, 0.5, 0.81], [-0.7, 0.2, 0.4], [0.1, -0.9, 0.3]]), dim=1)
    elif name == "two_chunks":              # M > 1 048 576 (two backward chunks, the second partial); m_pad >= 1e6: the lit fallback
        x, d = march(env, 256, 0.18)
        M = x.shape[0]
        assert M > CHUNK_TILES * 128, M
        cs.counter = torch.tensor([M, 0], dtype=torch.int32, device="cuda")
        cs.align, cs.cap, cs.m_pad = 128, M + 128 + 300, M + 128 - M % 128
    cs.M = M
    if cs.segs is None:
        cs.mpad = [cs.m_pad]
        lights = l0[None]
    cs.light = lights.float().cuda().contiguous()
    n_all = cs.cap + GUARD
    cs.x = torch.full((n_all, 3), float("nan"), device="cuda"); cs.x[:M] = x[:M]
    cs.d = torch.full((n_all, 3), float("nan"), device="cuda"); cs.d[:M] = d[:M]
    cs.noise = torch.from_numpy(np.random.default_rng(17).standard_normal((n_all, 3)).astype(np.float32)).cuda()
    env.cases[name] = cs
    return cs


def row_facts(cs, r0, r1):
    """F.Rows of rows [r0, r1) as the kernels see them (x of non-sample rows is 0)"""
    rows = torch.arange(r0, r1, device="cuda", dtype=torch.long)
    real = rows < cs.M
    in_range = rows < cs.m_pad
    x = torch.where(real[:, None], cs.x[r0:r1], 0.0)
    d = torch.where(real[:, None], cs.d[r0:r1], 0.0)
    if cs.segs is None:
        view = torch.zeros_like(rows)
        pad_idx = rows - cs.M
    else:
        b = torch.tensor(list(cs.segs_host.bounds)[:2 * cs.nv + 1], device="cuda")
        sgm = (rows[:, None] >= b[None, 1:2 * cs.nv]).sum(1)
        view = torch.where(sgm < cs.nv, sgm, sgm - cs.nv)
        pad_idx = rows - b[sgm]
    mpad = torch.tensor(cs.mpad, device="cuda")[view]
    return rows, x, d, real, in_range, view, pad_idx, mpad


def make_R(cs, r0, r1, n_evals, z_mode="inject"):
    rows, x, d, real, in_range, view, pad_idx, mpad = row_facts(cs, r0, r1)
    if n_evals > 7:
        if z_mode == "inject":
            z = cs.noise[r0:r1]
        else:
            z = F.smooth_z(rows, x, real, pad_idx, cs.seed, cs.noise_mode)
        xp = torch.where(in_range[:, None], F.perturbed(x, z), 0.0)
    else:
        xp = torch.zeros_like(x)
    return F.Rows(x, d, xp, in_range, real, view, mpad, cs.light.double()[view])


# ---------------------------------------------------------------------------------------------------------------------------
# kernel calls
# ---------------------------------------------------------------------------------------------------------------------------
def make_io(env, cs, noise, cache=None, cache_tiles=0, valid=0):
    io = env.L.FieldIO()
    io.xyzs, io.dirs = cs.x.data_ptr(), cs.d.data_ptr()
    io.counter = cs.counter.data_ptr() if cs.counter is not None else None
    io.m_fixed, io.align, io.cap = cs.m_fixed, cs.align, cs.cap
    io.smooth_noise = cs.noise.data_ptr() if noise else None
    io.seed, io.noise_mode = cs.seed, cs.noise_mode
    io.enc_cache = cache.data_ptr() if cache is not None else None
    io.enc_cache_tiles, io.enc_cache_valid = cache_tiles, valid
    io.segs = cs.segs.data_ptr() if cs.segs is not None else None
    io.n_views = cs.nv if cs.segs is not None else 0
    return io


def cfg(env, n_evals, shading, ratio, cs):
    c = env.L.FieldCfg()
    c.bound, c.blob_density, c.blob_radius = 1.0, 5.0, 0.1
    c.n_evals, c.shading, c.ambient_ratio = n_evals, env.L.SHADING[shading], ratio
    c.light_d = cs.light.data_ptr()
    return c


def run_fwd(env, W, cs, n_evals, shading, ratio, noise=True, cache_tiles=None):
    n_all = cs.cap + GUARD
    tiles = (cs.cap + 127) // 128
    cache_tiles = tiles if cache_tiles is None else cache_tiles
    o = SimpleNamespace(sig=canvas(n_all), rgb=canvas(n_all * 3), nrm=canvas(n_all * 3), tape=canvas(n_all * 16),
                        cache=canvas(cache_tiles * 13 * 128 * 32), losses=canvas(2 * cs.nv + 16), cache_tiles=cache_tiles,
                        n_evals=n_evals, shading=shading, ratio=ratio)
    partials = torch.zeros(2 * cs.nv * env.ctas, device="cuda")
    io = make_io(env, cs, noise, o.cache, cache_tiles)
    cf = cfg(env, n_evals, shading, ratio, cs)
    p = env.L.ptr
    env.L.check(env.lib.mi3d_field_forward(C.byref(io), p(W.table), C.byref(W.hg), C.byref(W.mlp), C.byref(cf), p(o.sig), p(o.rgb),
                                           p(o.nrm), p(o.tape), p(partials), C.c_void_p(o.losses.data_ptr()),
                                           C.c_void_p(o.losses.data_ptr() + 4 * cs.nv), env.L.stream()), "field_forward")
    torch.cuda.synchronize()
    return o


def base_grads(W):
    g = torch.Generator(device="cuda").manual_seed(5)
    table = (torch.rand(2 * W.n_entries, device="cuda", generator=g) - 0.5) * 2 ** -5
    mlp = [(torch.rand(t.shape, device="cuda", generator=g) - 0.5) * 2 ** -5 for t in W.ws]
    return table, mlp


def run_bwd(env, W, cs, o, up, variant, noise=True):
    """variant: 'cache' (every chunk from the forward's cache), 'partial' (a cache one tile short: re-gathered), 'nocache',
    'noworkspace' (the chain kernel gathers in-kernel)"""
    gt, gm = base_grads(W)
    gms = env.L.Mlp()
    for name, t in zip(("w1", "b1", "w2", "b2", "w3", "b3"), gm):
        setattr(gms, name, t.data_ptr())
    tiles = o.cache_tiles
    if variant == "cache":
        io = make_io(env, cs, noise, o.cache, tiles, 1)
    elif variant == "partial":
        io = make_io(env, cs, noise, o.cache, max(tiles - 1, 0), 1)
    else:
        io = make_io(env, cs, noise)
    cf = cfg(env, o.n_evals, o.shading, o.ratio, cs)
    p = env.L.ptr
    ws = None if variant == "noworkspace" else env.scratch
    env.L.check(env.lib.mi3d_field_backward(C.byref(io), p(W.table), C.byref(W.hg), C.byref(W.mlp), C.byref(cf), p(o.tape),
                                            p(up.get("gs")), p(up.get("gc")), p(up.get("gn")), p(up.get("go")), p(up.get("gl")),
                                            p(gt), C.byref(gms), p(ws), env.L.stream()), "field_backward")
    torch.cuda.synchronize()
    return gt, gm


def upstream(cs, kinds, seed=7, rows=None):
    """upstream gradients: gs / gc / gn [cap + GUARD] NaN past the sample count (and outside `rows` zero), go / gl per view"""
    g = torch.Generator(device="cuda").manual_seed(seed)
    n_all = cs.cap + GUARD
    up = {}
    for k, w in (("gs", 1), ("gc", 3), ("gn", 3)):
        if k in kinds:
            t = torch.randn(n_all, w, device="cuda", generator=g) * (0.1 if k == "gn" else 1.0)
            if rows is not None:
                keep = torch.zeros(n_all, dtype=torch.bool, device="cuda"); keep[rows[0]:rows[1]] = True
                t = torch.where(keep[:, None], t, 0.0)
            t[cs.M:] = float("nan")
            up[k] = t.reshape(-1).contiguous()
    if "go" in kinds:
        up["go"] = torch.tensor([3.0, 2.0, 4.0][:cs.nv], device="cuda")
    if "gl" in kinds:
        up["gl"] = torch.tensor([5.0, 7.0, 1.5][:cs.nv], device="cuda")
    if "gl0" in kinds:
        up["gl"] = torch.zeros(cs.nv, device="cuda")
    return up


# ---------------------------------------------------------------------------------------------------------------------------
# reference passes and checks
# ---------------------------------------------------------------------------------------------------------------------------
def check_forward(env, W, cs, o, name, z_mode="inject"):
    """every in-range row's outputs and tape, every cached encoding, the loss means; everything past the written rows untouched"""
    wst = Worst(name)
    f = W.f64
    nv, n_evals = cs.nv, o.n_evals
    t_o = torch.zeros(nv, dtype=torch.float64, device="cuda")
    e_o, t_s, e_s, m_o, m_s = t_o.clone(), t_o.clone(), t_o.clone(), t_o.clone(), t_o.clone()
    amb = 0
    # the forward caches the tiles it evaluates: those below min(cache_tiles, ceil(m_pad / 128)), all 128 rows of each
    ctiles = min(o.cache_tiles, (cs.m_pad + 127) // 128)
    end = max(ctiles * 128, cs.m_pad)
    cache = o.cache.view(-1, 13, 128, 32) if o.cache_tiles else None
    if cache is not None:
        untouched("enc_cache past the evaluated tiles", cache[ctiles:])
    for r0 in range(0, end, CHUNK):
        r1 = min(end, r0 + CHUNK)
        R = make_R(cs, r0, r1, n_evals, z_mode)
        ref = f.forward(R, n_evals, o.shading, o.ratio, keep_enc=cache is not None)
        amb += ref["amb_normal"]
        if cache is not None and r0 < ctiles * 128:
            c1 = min(r1, ctiles * 128)
            got = cache[r0 // 128:(c1 + 127) // 128].permute(0, 2, 1, 3).reshape(-1, 13, 32)[:c1 - r0]
            for e in range(n_evals):
                enc, ee = ref["encs"][e]
                wst.add("enc_cache", got[:, e], enc[:c1 - r0], ee[:c1 - r0])
            if n_evals < 13:
                untouched("enc_cache beyond n_evals", got[:, n_evals:])
        k = torch.arange(r0, r1, device="cuda") < cs.m_pad
        if not bool(k.any()):
            continue
        r1k = r0 + int(k.sum())
        sl = slice(0, r1k - r0)
        wst.add("sigma", o.sig[r0:r1k], ref["sigma"][sl], ref["e_sigma"][sl])
        wst.add("rgb", o.rgb.view(-1, 3)[r0:r1k], ref["rgb"][sl], ref["e_rgb"][sl])
        if n_evals >= 7:
            wst.add("normal", o.nrm.view(-1, 3)[r0:r1k], ref["normal"][sl], ref["e_normal"][sl])
        wst.add("tape", o.tape.view(-1, 16)[r0:r1k], ref["tape"][sl], ref["e_tape"][sl])
        view = R.view[sl]
        mp = R.mpad[sl].double()
        for v in range(nv):
            s = view == v
            t_o[v] += (ref["t_orient"][sl][s] / mp[s]).sum(); e_o[v] += (ref["e_orient"][sl][s] / mp[s]).sum()
            t_s[v] += (ref["t_smooth"][sl][s] / (3 * mp[s])).sum(); e_s[v] += (ref["e_smooth"][sl][s] / (3 * mp[s])).sum()
            m_o[v] += (ref["t_orient"][sl][s].abs() / mp[s]).sum(); m_s[v] += (ref["t_smooth"][sl][s].abs() / (3 * mp[s])).sum()
    for t in (o.sig[cs.m_pad:], o.rgb[3 * cs.m_pad:], o.nrm[3 * cs.m_pad:] if n_evals >= 7 else o.nrm, o.tape[16 * cs.m_pad:]):
        untouched(f"{name}: outputs past m_pad", t)
    tiles = (cs.m_pad + 127) // 128
    gam = ((tiles // env.ctas + 1) * 128 + 4 * env.ctas + 300) * F.U
    wst.add("loss_orient", o.losses[:nv], t_o, e_o + gam * m_o + 2 * F.U * t_o.abs())
    wst.add("loss_smooth", o.losses[nv:2 * nv], t_s, e_s + gam * m_s + 2 * F.U * t_s.abs())
    wst.done(ill_conditioned_normals=amb)
    assert amb <= AMB_MAX * cs.m_pad + 16          # the spliced face points may be among them


def ref_backward(env, W, cs, o, up, z_mode="inject"):
    f = W.f64
    acc = F.BwdAcc(W.n_entries, "cuda")
    amb_rows = 0
    n_evals = o.n_evals
    need_ptaps = "gl" in up and bool((up["gl"] != 0).any()) and n_evals > 7
    for r0 in range(0, cs.m_pad, CHUNK):
        r1 = min(cs.m_pad, r0 + CHUNK)
        R = make_R(cs, r0, r1, n_evals, z_mode)
        n = r1 - r0
        real = R.real
        z1 = torch.zeros(n, device="cuda", dtype=torch.float64)
        gs = torch.where(real, up["gs"][r0:r1].double(), 0.0) if "gs" in up else z1
        gc = torch.where(real[:, None], up["gc"].view(-1, 3)[r0:r1].double(), 0.0) if "gc" in up else z1[:, None].expand(n, 3)
        gn = torch.where(real[:, None], up["gn"].view(-1, 3)[r0:r1].double(), 0.0) if ("gn" in up and n_evals >= 7) \
            else z1[:, None].expand(n, 3)
        # the kernel divides in fp32: Go = g / mpad, Gs = g / (3 mpad)
        Go = (up["go"][R.view] / R.mpad.float()).double() if ("go" in up and n_evals >= 7) else z1
        Gs = (up["gl"][R.view] / (3 * R.mpad.float())).double() if ("gl" in up and n_evals > 7) else z1
        dh, edh, dtap, edtap, amb = F.out_grads(o.tape.view(-1, 16)[r0:r1], R, gs, gc, gn, Go, Gs, n_evals, o.shading, o.ratio,
                                                need_ptaps)
        amb_rows += amb
        for e in range(n_evals):
            if e == 0:
                dO, edO = dh, edh
            else:
                dO = torch.nn.functional.pad(dtap[:, e - 1:e], (0, 3))
                edO = torch.nn.functional.pad(edtap[:, e - 1:e], (0, 3))
            live = (dO != 0).any(-1) | (edO != 0).any(-1)
            if not bool(live.any()):
                continue
            p = F.eval_pos(e, R.x, R.xp, f.bound)
            F.backward_eval(f, acc, p[live], dO[live], edO[live])
    acc.amb_rows = amb_rows
    return acc


def check_backward(env, W, cs, acc, gt, gm, name, n_evals, one_hot=False):
    wst = Worst(name)
    bt, bm = base_grads(W)
    tref = bt.double().view(-1, 2) + acc.table
    tb = acc.t_err + (acc.t_cnt[:, None] + 8) * F.U * (acc.t_mag + bt.double().view(-1, 2).abs())
    none = acc.t_cnt == 0
    got = gt.view(-1, 2)
    n_changed = int((got[none].view(torch.int32) != bt.view(-1, 2)[none].view(torch.int32)).sum())
    assert n_changed == 0, f"{name}: {n_changed} table entries without a reference contribution changed"
    wst.add("grad_table", got, tref, tb)
    r = ((got.double() - tref).abs() / tb.clamp(min=1e-300)).max(-1).values
    i = int(r.argmax())
    print(f"  worst table entry {i}: count {int(acc.t_cnt[i])}, ref {tref[i].tolist()}, got {got[i].tolist()}, "
          f"sum|c| {acc.t_mag[i].tolist()}, propagated {acc.t_err[i].tolist()}")
    tiles = (cs.m_pad + 127) // 128
    iters = (tiles // env.S + 1) * n_evals
    for i, k in enumerate(("w1", "b1", "w2", "b2", "w3", "b3")):
        gam = (iters + 4 * env.S + 64) * F.U + (F.gamma_bwd(128) if k in ("w1", "w2") else 5 * F.U)
        wst.add(f"d{k}", gm[i], bm[i].double() + acc.w[k], acc.w_err[k] + gam * (acc.w_mag[k] + bm[i].double().abs()))
    wst.done(ambiguous_relu_units=acc.amb_units, units=acc.units, ambiguous_kink_rows=acc.amb_rows)
    assert acc.amb_units <= AMB_MAX * max(acc.units, 1)
    assert acc.amb_rows <= AMB_MAX * cs.m_pad + 1


# ---------------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------------
FWD = {}


def forward_checked(env, W, cs, key, n_evals, shading, ratio, **kw):
    k = (key, n_evals, shading, ratio)
    if k not in FWD:
        o = run_fwd(env, W, cs, n_evals, shading, ratio, **kw)
        check_forward(env, W, cs, o, f"forward {key} n_evals={n_evals} {shading}")
        FWD[k] = o
    return FWD[k]


@pytest.mark.parametrize("n_evals,shading,ratio", [(1, "albedo", 1.0), (7, "albedo", 1.0), (7, "lambertian", 0.1), (7, "textureless", 0.2),
                                                   (7, "normal", 0.1), (13, "lambertian", 0.1), (13, "textureless", 0.3)])
def test_forward_fixed_rows(env, n_evals, shading, ratio):
    """m_fixed rows, align 0, at most one 128-row tile per CTA: every shading and evaluation count; a second launch is bit-identical"""
    W, cs = weights(env, "unit"), layout(env, "fixed")
    o = run_fwd(env, W, cs, n_evals, shading, ratio)
    check_forward(env, W, cs, o, f"fixed n_evals={n_evals} {shading}")
    o2 = run_fwd(env, W, cs, n_evals, shading, ratio)
    for a, b in ((o.sig, o2.sig), (o.rgb, o2.rgb), (o.nrm, o2.nrm), (o.tape, o2.tape), (o.cache, o2.cache), (o.losses, o2.losses)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


BWD_COMBOS = {                        # forward shading, upstream gradients -> the evaluations the backward needs (bwd_plan's e_end)
    "sigmas_albedo_e1": ("albedo", 1.0, ("gs", "gc")),
    "rgbs_lambertian_e7": ("lambertian", 0.1, ("gs", "gc")),
    "normals_only_e7": ("albedo", 1.0, ("gn",)),
    "smooth_only_e13": ("albedo", 1.0, ("gl",)),
    "smooth_zero_e7": ("lambertian", 0.1, ("gc", "go", "gl0")),
    "all_e13": ("textureless", 0.2, ("gs", "gc", "gn", "go", "gl")),
}


@pytest.mark.parametrize("combo", list(BWD_COMBOS))
def test_backward_march_rows(env, combo):
    """ray-ordered samples of the march (device counter, align 128, about 2.5 tiles per CTA) with adversarial rows spliced in, a
    13-evaluation forward, and each upstream combination through all four encoding sources"""
    W, cs = weights(env, "unit"), layout(env, "march")
    shading, ratio, kinds = BWD_COMBOS[combo]
    o = forward_checked(env, W, cs, "march", 13, shading, ratio)
    up = upstream(cs, kinds)
    acc = ref_backward(env, W, cs, o, up)
    for variant in ("cache", "partial", "nocache", "noworkspace"):
        gt, gm = run_bwd(env, W, cs, o, up, variant)
        check_backward(env, W, cs, acc, gt, gm, f"march {combo} {variant}", 13)


@pytest.mark.parametrize("which", ["second_tile_of_a_cta", "last_partial_tile"])
def test_backward_one_hot_tile(env, which):
    """g_sigmas / g_rgbs non-zero on one tile only: every table entry outside that tile's contributions stays bit-unchanged"""
    W, cs = weights(env, "unit"), layout(env, "march")
    o = forward_checked(env, W, cs, "march", 13, "lambertian", 0.1)
    tiles = (cs.m_pad + 127) // 128
    t = env.S + 3 if which == "second_tile_of_a_cta" else tiles - 1
    assert t < tiles
    up = upstream(cs, ("gs", "gc"), rows=(t * 128, (t + 1) * 128))
    acc = ref_backward(env, W, cs, o, up)
    for variant in ("cache", "noworkspace"):
        gt, gm = run_bwd(env, W, cs, o, up, variant)
        check_backward(env, W, cs, acc, gt, gm, f"one-hot tile {t} ({which}) {variant}", 13)


def test_rows_past_capacity_hash15(env):
    """counter[0] > cap with cap % 128 != 0 (no zero rows fit), on a hash grid of 2^15 entries per level (more hashed levels and
    collisions)"""
    W, cs = weights(env, "hash15"), layout(env, "over_cap")
    assert cs.counter[0] > cs.cap and cs.cap % 128 != 0
    o = run_fwd(env, W, cs, 13, "textureless", 0.2)
    check_forward(env, W, cs, o, "over_cap hash15")
    up = upstream(cs, ("gs", "gc", "go", "gl"))
    acc = ref_backward(env, W, cs, o, up)
    for variant in ("cache", "nocache", "noworkspace"):
        gt, gm = run_bwd(env, W, cs, o, up, variant)
        check_backward(env, W, cs, acc, gt, gm, f"over_cap hash15 {variant}", 13)


def test_two_backward_chunks(env):
    """M > 1 048 576 samples from a 256^2 camera: chunk 1 reads the forward's cache (8192 tiles, like the render workspace), chunk 2 is
    gathered; m_pad >= 1e6 selects the lit fallback (rgb = albedo); a one-hot gradient on the first tile of chunk 2"""
    W, cs = weights(env, "golden"), layout(env, "two_chunks")
    o = run_fwd(env, W, cs, 7, "lambertian", 0.1, cache_tiles=CHUNK_TILES)
    check_forward(env, W, cs, o, "two_chunks")
    a = o.rgb.view(-1, 3)[:cs.m_pad]
    assert torch.equal(a, o.tape.view(-1, 16)[:cs.m_pad, 1:4])          # lit fallback: colour = albedo
    up = upstream(cs, ("gs", "gc"))
    acc = ref_backward(env, W, cs, o, up)
    for variant in ("cache", "nocache"):
        gt, gm = run_bwd(env, W, cs, o, up, variant)
        check_backward(env, W, cs, acc, gt, gm, f"two_chunks {variant}", 7)
    t = CHUNK_TILES
    up = upstream(cs, ("gs", "gc"), rows=(t * 128, (t + 1) * 128))
    acc = ref_backward(env, W, cs, o, up)
    gt, gm = run_bwd(env, W, cs, o, up, "cache")
    check_backward(env, W, cs, acc, gt, gm, "two_chunks one-hot first tile of chunk 2", 7)


def test_multiview_segments(env):
    """3 views with uneven counts and one light each; zero rows after all views, view 2's owned by another rank (empty pad segment,
    mpad[2] above the local count); per-view loss means and loss gradients"""
    W, cs = weights(env, "unit"), layout(env, "multiview")
    o = run_fwd(env, W, cs, 13, "lambertian", 0.1)
    check_forward(env, W, cs, o, "multiview")
    up = upstream(cs, ("gs", "gc", "go", "gl"))
    acc = ref_backward(env, W, cs, o, up)
    for variant in ("cache", "nocache", "noworkspace"):
        gt, gm = run_bwd(env, W, cs, o, up, variant)
        check_backward(env, W, cs, acc, gt, gm, f"multiview {variant}", 13)


@pytest.mark.parametrize("name,mode", [("march", 0), ("multiview", 1)])
def test_philox_perturbation(env, name, mode):
    """noise_mode 0 (keyed by row) and 1 (by the position's float bits; zero rows by their index among the view's zero rows): the
    in-kernel draw against the fp64 restatement of Philox4x32-10 / Box-Muller.  cospif / sinpif / logf leave a few ulps on z that
    move a perturbed position by up to one fp32 ulp, which the element-wise bounds do not model; so the kernel's Philox run is held
    to the same kernels fed the restated draw: perturbed tap densities within 1e-3 relative, table and weight gradients within 1e-3
    of (|entry| + 1e-3 max), and no entry that only one of the two runs touches above 1e-7 of the largest entry (a one-ulp shift
    crossing a cell boundary puts a weight of ~ulp * scale there; a wrong key moves a perturbed position by ~0.01)"""
    W = weights(env, "unit")
    cs = layout(env, name)
    cs.noise_mode = mode
    keep = cs.noise
    try:
        o_p = run_fwd(env, W, cs, 13, "lambertian", 0.1, noise=False)
        z_all = torch.zeros(cs.cap + GUARD, 3, device="cuda")
        for r0 in range(0, cs.m_pad, CHUNK):
            r1 = min(cs.m_pad, r0 + CHUNK)
            rows, x, d, real, in_range, view, pad_idx, mpad = row_facts(cs, r0, r1)
            z_all[r0:r1] = F.smooth_z(rows, x, real, pad_idx, cs.seed, mode)
        cs.noise = z_all
        o_i = run_fwd(env, W, cs, 13, "lambertian", 0.1, noise=True)
        tp, ti = o_p.tape.view(-1, 16)[:cs.m_pad, 10:16].double(), o_i.tape.view(-1, 16)[:cs.m_pad, 10:16].double()
        rel = float(((tp - ti).abs() / ti.abs().clamp(min=1e-6)).max())
        up = upstream(cs, ("gc", "go", "gl"))
        gp, mp = run_bwd(env, W, cs, o_p, up, "cache", noise=False)
        gi, mi = run_bwd(env, W, cs, o_i, up, "cache", noise=True)
        bt = base_grads(W)[0]
        gmax = float((gi - bt).abs().max())
        tab = float(((gp - gi).abs() / (1e-3 * (gi - bt).abs() + 1e-3 * gmax)).max())
        # entries one run touches and the other does not: only the near-zero weights of a cell boundary crossed by a one-ulp
        # difference of the perturbed position may land there
        moved = (gp != bt) ^ (gi != bt)
        stray = float(torch.maximum((gp - bt).abs(), (gi - bt).abs())[moved].max()) / gmax if bool(moved.any()) else 0.0
        wr = max(float(((a - b).abs() / (1e-3 * (b.abs() + float(b.abs().max()) * 1e-3))).max()) for a, b in zip(mp, mi))
        print(f"\n[philox noise_mode={mode} {name}] tap rel {rel:.3g}, table ratio {tab:.3g}, weight ratio {wr:.3g}, "
              f"entries touched by one run only: {int(moved.sum())}, largest {stray:.3g} of max")
        assert rel < 1e-3 and tab <= 1.0 and wr <= 1.0 and stray < 1e-7
    finally:
        cs.noise_mode, cs.noise = 0, keep


def test_density_grid_refresh_all_cells(env):
    """mi3d_density_grid_update's sigma for all 128^3 cells (k_field_fwd, fp32 FFMA), with the cell jitter injected and a zero grid
    (grid = max(0 * decay, sigma) = sigma), against fp64: cell positions replicated in fp32 (fma of the jitter term), encodings
    16 u, layers (K + 2) u of |W| |x| + |b| per sequential fp32 FFMA chain"""
    W = weights(env, "golden")
    H = 128
    n = H ** 3
    jitter = torch.from_numpy(np.random.default_rng(21).random((1, n, 3), dtype=np.float32)).cuda()
    grid = torch.zeros(1, n, device="cuda")
    bits = torch.zeros(n // 8, dtype=torch.uint8, device="cuda")
    mean = torch.zeros(1, device="cuda")
    ws = torch.empty(env.lib.mi3d_density_grid_workspace_bytes(C.c_uint32(1), C.c_uint32(H)), dtype=torch.uint8, device="cuda")
    cf = env.L.FieldCfg()
    cf.bound, cf.blob_density, cf.blob_radius, cf.n_evals, cf.shading, cf.ambient_ratio = 1.0, 5.0, 0.1, 1, 0, 1.0
    p = env.L.ptr
    env.L.check(env.lib.mi3d_density_grid_update(p(grid), p(bits), C.c_uint32(1), C.c_uint32(H), C.c_float(1.0), C.c_float(0.95),
                                                 C.c_float(10.0), p(W.table), C.byref(W.hg), C.byref(W.mlp), C.byref(cf), p(jitter),
                                                 C.c_uint64(0), p(mean), p(ws), env.L.stream()), "density_grid_update")
    torch.cuda.synchronize()
    m = torch.arange(n, device="cuda", dtype=torch.long)

    def compact3(v):
        v = v & 0x49249249
        v = (v | (v >> 2)) & 0xC30C30C3
        v = (v | (v >> 4)) & 0x0F00F00F
        v = (v | (v >> 8)) & 0xFF0000FF
        return (v | (v >> 16)) & 0x0000FFFF
    c = torch.stack([compact3(m), compact3(m >> 1), compact3(m >> 2)], 1).float()
    hg_ = torch.tensor(1.0 / H, dtype=torch.float32)
    base = (2 * c) / torch.tensor(float(H - 1), dtype=torch.float32) - 1
    v1 = base * (torch.tensor(1.0, dtype=torch.float32) - hg_)
    xyz = ((jitter[0] * 2 - 1).double() * float(hg_) + v1.double()).float()          # fmaf((u*2-1), half_grid, v)
    wst = Worst("density grid 128^3")
    f = W.f64
    m_ = f.mlp
    fw = lambda K: (K + 2) * F.U
    for r0 in range(0, n, 4 * CHUNK):
        pch = xyz[r0:r0 + 4 * CHUNK]
        u = F.to_u(pch, 1.0)
        enc, e_enc, _ = f.grid.encode(u)
        z1 = enc @ m_.w[0].T + m_.b[0]
        e1 = e_enc @ m_.a[0].T + fw(32) * ((enc.abs() + e_enc) @ m_.a[0].T + m_.b[0].abs())
        h1 = z1.clamp(min=0)
        z2 = h1 @ m_.w[1].T + m_.b[1]
        e2 = e1 @ m_.a[1].T + fw(64) * ((h1 + e1) @ m_.a[1].T + m_.b[1].abs())
        h2 = z2.clamp(min=0)
        o0 = h2 @ m_.w[2][0] + m_.b[2][0]
        eo = e2 @ m_.a[2][0] + fw(64) * ((h2 + e2) @ m_.a[2][0] + m_.b[2][0].abs())
        pd = pch.double()
        dd = (pd * pd).sum(-1)
        blob = f.blob_density * torch.exp(-dd / f.two_r2)
        arg = o0 + blob
        e_arg = eo + blob * (3 * F.U * dd / f.two_r2 + 5 * F.U) + F.U * arg.abs()
        sig = torch.exp(arg)
        wst.add("sigma", grid[0, r0:r0 + 4 * CHUNK], sig, sig * (torch.expm1(e_arg) + 3 * F.U))
    wst.done()
