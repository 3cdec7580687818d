"""tests/field_ref64.py -- TEST INFRASTRUCTURE: an fp64 restatement of the fused field kernels (csrc/field.cu) with error bounds.

What k_field_fwd_tc / k_field_bwd_tc compute per marched sample (nerf/network_tcnn.py:94-170, nerf/renderer.py:513-524), in torch
float64 on whatever device the tensors live on, chunk by chunk:

* Positions are the kernels' fp32 decisions, replicated exactly: the smoothing perturbation xp = fma(z, 0.01f, x), the finite-difference
  tap p[axis] += +-0.01f with ALL three coordinates then clamped to +-bound, u = (p + b) / (2b) in fp32, cell and fraction from
  fmaf(scale, u, 0.5f) (one fp64 operation, like oracle/field_ref.HashGridRef), and hg_index for dense levels (with the wrap at the upper
  face) and hashed levels.  From there every value is fp64.
* The in-kernel perturbation (mi3d_philox = Philox4x32-10, mi3d_u01, gauss_pair, gauss_pos) in uint32 arithmetic on int64 tensors.
  cospif / sinpif / logf carry a few ulps the restatement cannot reproduce, so `smooth_z` returns the fp32-rounded fp64 value.
* Every computed quantity X comes with a bound E_X on |kernel - X| ("magnitude pass": the same formulas on absolute values, times the
  rounding the kernel's arithmetic applies, plus the propagated input error).  u = 2^-24 is one fp32 rounding;
    forward layer GEMMs, 3-term tf32 split on wgmma:  per product 3 * 2^-22, plus 2 u per add over 3 K adds   (gamma_fwd)
    backward layer GEMMs, 6-term bf16 split:          per product 2^-21,     plus 2 u per add over 6 K adds   (gamma_bwd)
    owner fp32 arithmetic (normals, shading, losses): a stated small multiple of u of the magnitude.
  The backward reference starts from the kernel's own forward tape (sigma0, albedo, 12 tap densities: checked against this reference's
  forward separately), so its bounds carry only the backward's own arithmetic and the encodings' error.
* Kinks (ReLU pre-activations, the ndl clamp at 0.1, sign(df) of the smoothness term, the ndd > 0 test) whose fp64 margin lies inside
  the bound admit both branches: the bound grows by the size of the jump, and the number of such units is returned so that callers
  can fail when too many checks would become loose.
"""
import math

import torch

U = 2.0 ** -24
MASK32 = 0xFFFFFFFF
PRIME_Y, PRIME_Z = 2654435761, 805459861
E15 = 3269017.372472110639                 # exp(15): trunc_exp's gradient clamp (activation.py:12-16)
EPS32 = float(torch.tensor(1e-2, dtype=torch.float32))
SHADING = {"albedo": 0, "lambertian": 1, "textureless": 2, "normal": 3}


def gamma_fwd(K):
    return 3 * 2.0 ** -22 + 6 * K * U


def gamma_bwd(K):
    return 2.0 ** -21 + 12 * K * U


# ---------------------------------------------------------------------------------------------------------------------------
# Philox4x32-10 and the Gaussian draws of the smoothness perturbation (mi3d_common.cuh, field.cu gauss_pair / gauss_pos)
# ---------------------------------------------------------------------------------------------------------------------------
def _mulhilo(m, a):
    a1, a0 = a >> 16, a & 0xFFFF
    s, t = m * a1, m * a0
    lo = (((s & 0xFFFF) << 16) + t) & MASK32
    hi = (s + (t >> 16)) >> 16
    return hi, lo


def philox(c, key):
    """c: 4 int64 tensors holding uint32 counters; key: (k0, k1) python ints"""
    c0, c1, c2, c3 = c
    k0, k1 = key
    for _ in range(10):
        hi0, lo0 = _mulhilo(0xD2511F53, c0)
        hi1, lo1 = _mulhilo(0xCD9E8D57, c2)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + 0x9E3779B9) & MASK32, (k1 + 0xBB67AE85) & MASK32
    return c0, c1, c2, c3


def _u01(v):
    return (v >> 8).double() * 2.0 ** -24


def _gauss(r):
    u1, u2 = _u01(r[0]).clamp(min=2.0 ** -24), _u01(r[1])
    u3, u4 = _u01(r[2]).clamp(min=2.0 ** -24), _u01(r[3])
    m1, m2 = torch.sqrt(-2 * torch.log(u1)), torch.sqrt(-2 * torch.log(u3))
    return torch.stack([m1 * torch.cos(2 * math.pi * u2), m1 * torch.sin(2 * math.pi * u2), m2 * torch.cos(2 * math.pi * u4)], -1).float()


def gauss_pair(seed, idx, salt):
    z = torch.zeros_like(idx)
    r = philox((idx & MASK32, z + salt, z, z + 0x736D6F6F), (seed & MASK32, (seed >> 32) & MASK32))
    return _gauss(r)


def gauss_pos(seed, x):
    bits = x.contiguous().view(torch.int32).long() & MASK32
    r = philox((bits[:, 0], bits[:, 1], bits[:, 2], torch.full_like(bits[:, 0], 0x706F7321)), (seed & MASK32, (seed >> 32) & MASK32))
    return _gauss(r)


def smooth_z(rows, x, real, pad_idx, seed, noise_mode):
    """z ~ N(0,1)^3 of rows (int64) as the kernels draw it in-kernel (smooth_z in field.cu): noise_mode 0 keys by row; noise_mode 1 by
    the float bits of the position for samples and by the index among the view's zero rows for zero rows"""
    if noise_mode == 0:
        return gauss_pair(seed, rows, 1)
    z = gauss_pair(seed, pad_idx.clamp(min=0), 2)
    if bool(real.any()):
        z[real] = gauss_pos(seed, x[real])
    return z


# ---------------------------------------------------------------------------------------------------------------------------
# positions and the hash grid
# ---------------------------------------------------------------------------------------------------------------------------
def perturbed(x, z):
    """xp = fmaf(z, 0.01f, x) (fp32; the product is exact in fp64)"""
    return (z.double() * EPS32 + x.double()).float()


def eval_pos(e, x, xp, bound):
    p = (xp if e >= 7 else x).clone()
    if e > 0:
        t = (e - 1) % 6
        axis, sgn = t >> 1, (-EPS32 if t & 1 else EPS32)
        p[:, axis] = p[:, axis] + torch.tensor(sgn, dtype=torch.float32)
        p = p.clamp(-bound, bound)
    return p


def to_u(p, bound):
    b = torch.tensor(bound, dtype=torch.float32)
    return (p + b) / (2 * b)


class Grid:
    """level geometry of an mi3d_hashgrid (offsets / sizes / ress / scales) and the fp64 table"""

    def __init__(self, offsets, sizes, ress, scales, table):
        self.L = len(offsets)
        self.offsets, self.sizes, self.ress = [int(v) for v in offsets], [int(v) for v in sizes], [int(v) for v in ress]
        self.scales = [float(torch.tensor(float(s), dtype=torch.float32)) for s in scales]
        self.hashed = [r ** 3 > s for r, s in zip(self.ress, self.sizes)]
        self.table = table.double().view(-1, 2)

    @classmethod
    def from_struct(cls, hg, table):
        n = hg.n_levels
        return cls(hg.offsets[:n], hg.sizes[:n], hg.ress[:n], hg.scales[:n], table)

    def corners(self, u, l):
        """entry index [n,8] (int64) and trilinear weight [n,8] (fp64, from the fp32 fractions) of level l at positions u [n,3] fp32"""
        pos = (u.double() * self.scales[l] + 0.5).float()
        fl = torch.floor(pos)
        w = (pos - fl).double()
        c = fl.long() & MASK32
        size, res = self.sizes[l], self.ress[l]
        idx, wt = [], []
        for corner in range(8):
            cc = [(c[:, d] + ((corner >> d) & 1)) & MASK32 for d in range(3)]
            ww = torch.ones_like(w[:, 0])
            for d in range(3):
                ww = ww * (w[:, d] if (corner >> d) & 1 else 1 - w[:, d])
            if self.hashed[l]:
                i = cc[0] ^ ((cc[1] * PRIME_Y) & MASK32) ^ ((cc[2] * PRIME_Z) & MASK32)
                i = i & (size - 1) if size & (size - 1) == 0 else i % size
            else:
                i = (cc[0] + cc[1] * res + cc[2] * res * res) & MASK32
                i = torch.where(i >= size, i % size, i)
            idx.append(i + self.offsets[l])
            wt.append(ww)
        return torch.stack(idx, 1), torch.stack(wt, 1)

    def encode(self, u):
        """encodings [n,32] fp64, their bound [n,32], and the corners of every level (for the scatter)"""
        enc, mag, cs = [], [], []
        for l in range(self.L):
            idx, wt = self.corners(u, l)
            v = self.table[idx]                                    # [n,8,2]
            enc.append((wt[..., None] * v).sum(1))
            mag.append((wt[..., None] * v.abs()).sum(1))
            cs.append((idx, wt))
        enc, mag = torch.cat(enc, 1), torch.cat(mag, 1)
        return enc, 16 * U * mag, cs


class Mlp:
    def __init__(self, w1, b1, w2, b2, w3, b3):
        self.w = [t.double() for t in (w1, w2, w3)]
        self.b = [t.double() for t in (b1, b2, b3)]
        self.a = [t.abs() for t in self.w]


def layers(m, enc, e_enc, gamma):
    """z1, h1, z2, h2, o (no output bias) with bounds; gamma(K) is the GEMM's relative rounding"""
    d1 = enc @ m.w[0].T
    z1 = d1 + m.b[0]
    e1 = e_enc @ m.a[0].T + gamma(32) * ((enc.abs() + e_enc) @ m.a[0].T) + U * (z1.abs() + m.b[0].abs())
    h1 = z1.clamp(min=0)
    d2 = h1 @ m.w[1].T
    z2 = d2 + m.b[1]
    e2 = e1 @ m.a[1].T + gamma(64) * ((h1 + e1) @ m.a[1].T) + U * z2.abs()
    h2 = z2.clamp(min=0)
    o = h2 @ m.w[2].T
    eo = e2 @ m.a[2].T + gamma(64) * ((h2 + e2) @ m.a[2].T)
    return dict(z1=z1, e1=e1, h1=h1, z2=z2, e2=e2, h2=h2, o=o, eo=eo)


# ---------------------------------------------------------------------------------------------------------------------------
# forward
# ---------------------------------------------------------------------------------------------------------------------------
class Rows:
    """per-row facts of one chunk: x / d (fp32, zero for non-sample rows), xp (fp32), in_range / real masks, view, mpad, light [n,3]"""

    def __init__(self, x, d, xp, in_range, real, view, mpad, light):
        self.x, self.d, self.xp, self.in_range, self.real = x, d, xp, in_range, real
        self.view, self.mpad, self.light = view, mpad, light
        self.n = x.shape[0]


def _normal(sp, sn, esp, esn):
    g = -(0.5 * (sp - sn) / EPS32)
    eg = 0.5 / EPS32 * (esp + esn + 3 * U * (sp - sn).abs())
    S = (g * g).sum(-1, keepdim=True)
    q = S.clamp(1e-20, 1e32)
    n = g / q.sqrt()
    en = (2 * (eg * eg).sum(-1, keepdim=True).sqrt() / S.sqrt().clamp(min=1e-300) + 4 * U).clamp(max=2.0).expand_as(n)
    return n, en, S


class Field64:
    def __init__(self, grid, mlp, bound=1.0, blob_density=5.0, blob_radius=0.1):
        self.grid, self.mlp = grid, mlp
        self.bound = float(torch.tensor(bound, dtype=torch.float32))
        self.blob_density = float(torch.tensor(blob_density, dtype=torch.float32))
        r = float(torch.tensor(blob_radius, dtype=torch.float32))
        self.two_r2 = float(torch.tensor(2.0 * r * r, dtype=torch.float32))

    def eval_point(self, p, gamma=gamma_fwd):
        """sigma / albedo (fp64) with bounds at fp32 positions p [n,3], plus the encodings and layer values"""
        u = to_u(p, self.bound)
        enc, e_enc, cs = self.grid.encode(u)
        a = layers(self.mlp, enc, e_enc, gamma)
        pd = p.double()
        dd = (pd * pd).sum(-1)
        blob = self.blob_density * torch.exp(-dd / self.two_r2)
        e_blob = blob * (3 * U * dd / self.two_r2 + 4 * U)
        h0 = a["o"][:, 0] + self.mlp.b[2][0]
        arg = h0 + blob
        e_arg = a["eo"][:, 0] + 2 * U * (h0.abs() + blob + arg.abs()) + e_blob
        sigma = torch.exp(arg)
        e_sigma = sigma * (torch.expm1(e_arg) + 3 * U)
        hc = a["o"][:, 1:] + self.mlp.b[2][1:]
        alb = torch.sigmoid(hc)
        e_alb = alb * (1 - alb) * (a["eo"][:, 1:] + U * hc.abs()) * (1 + 1e-3) + 4 * U * alb
        return dict(sigma=sigma, e_sigma=e_sigma, alb=alb, e_alb=e_alb, enc=enc, e_enc=e_enc, cs=cs, layers=a)

    def forward(self, R, n_evals, shading, ratio, keep_enc=False):
        """outputs of every row of R: sigma, rgb, normal, tape[16] and the loss terms, each with its bound"""
        n = R.n
        dev = R.x.device
        encs = []
        taps = torch.zeros(n, 12, dtype=torch.float64, device=dev)
        etaps = torch.zeros_like(taps)
        sigma0 = alb = None
        for e in range(n_evals):
            p = eval_pos(e, R.x, R.xp, self.bound)
            r = self.eval_point(p)
            if keep_enc:
                encs.append((r["enc"], r["e_enc"]))
            if e == 0:
                sigma0, es0, alb, ealb = r["sigma"], r["e_sigma"], r["alb"], r["e_alb"]
            else:
                taps[:, e - 1], etaps[:, e - 1] = r["sigma"], r["e_sigma"]
        out = dict(sigma=sigma0, e_sigma=es0, rgb=alb.clone(), e_rgb=ealb.clone(), encs=encs, amb_normal=0)
        tape = torch.cat([sigma0[:, None], alb, taps], 1)
        e_tape = torch.cat([es0[:, None], ealb, etaps], 1)
        out.update(tape=tape, e_tape=e_tape)
        t_o = torch.zeros(n, dtype=torch.float64, device=dev)
        e_to, t_s, e_ts = t_o.clone(), t_o.clone(), t_o.clone()
        if n_evals >= 7:
            nm, en, S = _normal(taps[:, 0:6:2], taps[:, 1:6:2], etaps[:, 0:6:2], etaps[:, 1:6:2])
            out.update(normal=nm, e_normal=en, amb_normal=int(((en > 0.05).any(-1) & R.in_range).sum()))
            lit = (SHADING[shading] != 0) & (R.mpad < 1000000)
            if shading != "albedo" and bool(lit.any()):
                l = R.light
                ndl = (nm * l).sum(-1)
                endl = (en * l.abs()).sum(-1) + 3 * U * (nm * l).abs().sum(-1)
                lam = ratio + (1 - ratio) * ndl.clamp(min=0.1)
                elam = (1 - ratio) * endl + 3 * U * lam.abs()
                if shading == "textureless":
                    col, ecol = lam[:, None].expand(n, 3), elam[:, None].expand(n, 3)
                elif shading == "normal":
                    col, ecol = (nm + 1) / 2, en / 2 + 2 * U
                else:
                    col = alb * lam[:, None]
                    ecol = alb * elam[:, None] + lam[:, None].abs() * ealb + U * col.abs()
                out["rgb"] = torch.where(lit[:, None], col, out["rgb"])
                out["e_rgb"] = torch.where(lit[:, None], ecol, out["e_rgb"])
            wgt = 1 - torch.exp(-sigma0)
            e_wgt = torch.exp(-sigma0) * torch.expm1(es0) + 3 * U
            dd = (nm * R.d.double()).sum(-1)
            ndd = dd.clamp(min=0)
            endd = (en * R.d.double().abs()).sum(-1) + 3 * U * (nm * R.d.double()).abs().sum(-1)
            t_o = wgt * ndd * ndd
            e_to = wgt * (2 * ndd * endd + endd * endd) + ndd * ndd * e_wgt + 3 * U * t_o
            if n_evals > 7:
                npn, enp, _ = _normal(taps[:, 6:12:2], taps[:, 7:12:2], etaps[:, 6:12:2], etaps[:, 7:12:2])
                t_s = (nm - npn).abs().sum(-1)
                e_ts = (en + enp).sum(-1) + 4 * U * (nm.abs() + npn.abs()).sum(-1)
        keep = R.in_range.double()
        out.update(t_orient=t_o * keep, e_orient=e_to * keep, t_smooth=t_s * keep, e_smooth=e_ts * keep)
        return out


# ---------------------------------------------------------------------------------------------------------------------------
# backward
# ---------------------------------------------------------------------------------------------------------------------------
C_OWN = 64          # owner fp32 arithmetic of sample_out_grads: bound = C_OWN u of the magnitude pass


def _normal_bwd(g, dn, edn, mdn):
    """d/dg of n = safe_normalize(g) given d/dn (value, bound of its error, magnitude)"""
    S = (g * g).sum(-1, keepdim=True)
    inside = ((S >= 1e-20) & (S <= 1e32)).double()
    inv = 1 / S.clamp(1e-20, 1e32).sqrt()
    dot = (dn * g).sum(-1, keepdim=True)
    dg = dn * inv - (dot * inv ** 3) * g * inside
    ga = g.abs()
    mag = mdn * inv + ((mdn * ga).sum(-1, keepdim=True) * inv ** 3) * ga
    err = edn * inv + ((edn * ga).sum(-1, keepdim=True) * inv ** 3) * ga + C_OWN * U * mag
    return dg, err, mag


def out_grads(tape, R, gs, gc, gn, Go, Gs, n_evals, shading, ratio, need_ptaps):
    """sample_out_grads (field.cu) in fp64 from the kernel's tape [n,16] (fp32): dO of evaluation 0 [n,4] and of the 12 taps [n,12],
    with bounds, and the number of rows where a kink lies inside the bound"""
    t = tape.double()
    n = t.shape[0]
    sigma0, alb, taps = t[:, 0], t[:, 1:4], t[:, 4:16]
    gs, gc = gs.double(), gc.double()
    dalb, edalb = gc.clone(), torch.zeros_like(gc)
    dtap, edtap = torch.zeros_like(taps), torch.zeros_like(taps)
    amb = torch.zeros(n, dtype=torch.bool, device=t.device)
    en = 16 * U                                         # |n_kernel - n| on the same tape (unit vector)
    if n_evals >= 7:
        sp, sn = taps[:, 0:6:2], taps[:, 1:6:2]
        g = -(0.5 * (sp - sn) / EPS32)
        nm = g / (g * g).sum(-1, keepdim=True).clamp(1e-20, 1e32).sqrt()
        dn = gn.double().clone()
        mdn = dn.abs()
        edn = torch.zeros_like(dn)
        lit = (SHADING[shading] != 0) & (R.mpad < 1000000)
        if shading != "albedo":
            l = R.light
            ndl = (nm * l).sum(-1)
            lam = ratio + (1 - ratio) * ndl.clamp(min=0.1)
            if shading == "textureless":
                dlam, mdlam = gc.sum(-1), gc.abs().sum(-1)
                dalb_l = torch.zeros_like(gc)
            elif shading == "normal":
                dlam, mdlam = torch.zeros_like(lam), torch.zeros_like(lam)
                dalb_l = torch.zeros_like(gc)
                dn = dn + torch.where(lit[:, None], 0.5 * gc, 0.0)
                mdn = mdn + torch.where(lit[:, None], 0.5 * gc.abs(), 0.0)
            else:
                dlam, mdlam = (gc * alb).sum(-1), (gc * alb).abs().sum(-1)
                dalb_l = gc * lam[:, None]
            margin = ndl - 0.1
            kink = lit & (margin.abs() <= en * l.abs().sum(-1) + 4 * U)
            amb |= kink & (mdlam != 0)
            on = (lit & (margin >= 0)).double()[:, None]
            k = (dlam * (1 - ratio))[:, None]
            dn = dn + on * k * l
            mdn = mdn + on * k.abs() * l.abs()
            edn = edn + kink.double()[:, None] * k.abs() * l.abs()
            dalb = torch.where(lit[:, None], dalb_l, dalb)
            # lam of the kernel (its own n) differs by (1 - ratio) |l| en; the clamp is 1-Lipschitz
            edalb = torch.where(lit[:, None], gc.abs() * ((1 - ratio) * en * l.abs().sum(-1) + 4 * U * lam.abs())[:, None], edalb)
        Gor = Go.double()
        wgt = 1 - torch.exp(-sigma0)
        ndd = (nm * R.d.double()).sum(-1)
        on = (ndd > 0).double()[:, None]
        k = (Gor * wgt * 2 * ndd)[:, None]
        dn = dn + on * k * R.d.double()
        mdn = mdn + on * k.abs() * R.d.double().abs()
        edn = edn + (Gor.abs() * wgt * 2 * (en * R.d.double().abs().sum(-1) + 4 * U))[:, None] * R.d.double().abs()
        dnp = torch.zeros_like(dn)
        mdnp, ednp = torch.zeros_like(dn), torch.zeros_like(dn)
        if need_ptaps:
            sp2, sn2 = taps[:, 6:12:2], taps[:, 7:12:2]
            g2 = -(0.5 * (sp2 - sn2) / EPS32)
            npn = g2 / (g2 * g2).sum(-1, keepdim=True).clamp(1e-20, 1e32).sqrt()
            df = nm - npn
            sg = torch.sign(df)
            Gsd = Gs.double()[:, None]
            dn, dnp = dn + Gsd * sg, dnp - Gsd * sg
            mdn, mdnp = mdn + Gsd.abs() * sg.abs(), mdnp + Gsd.abs() * sg.abs()
            kink = (df.abs() <= 2 * en) & (Gsd != 0)
            amb |= kink.any(-1)
            edn, ednp = edn + 2 * Gsd.abs() * kink, ednp + 2 * Gsd.abs() * kink
        edn = edn + C_OWN * U * mdn
        dg, edg, mdg = _normal_bwd(g, dn, edn, mdn)
        m = taps[:, 0:6].clamp(max=E15)
        k = 0.5 / EPS32
        dtap[:, 0:6:2], dtap[:, 1:6:2] = -k * dg * m[:, 0::2], k * dg * m[:, 1::2]
        edtap[:, 0:6:2] = k * (edg + C_OWN * U * mdg) * m[:, 0::2]
        edtap[:, 1:6:2] = k * (edg + C_OWN * U * mdg) * m[:, 1::2]
        if need_ptaps:
            ednp = ednp + C_OWN * U * mdnp
            dg2, edg2, mdg2 = _normal_bwd(g2, dnp, ednp, mdnp)
            m2 = taps[:, 6:12].clamp(max=E15)
            dtap[:, 6:12:2], dtap[:, 7:12:2] = -k * dg2 * m2[:, 0::2], k * dg2 * m2[:, 1::2]
            edtap[:, 6:12:2] = k * (edg2 + C_OWN * U * mdg2) * m2[:, 0::2]
            edtap[:, 7:12:2] = k * (edg2 + C_OWN * U * mdg2) * m2[:, 1::2]
    dh = torch.zeros(n, 4, dtype=torch.float64, device=t.device)
    edh = torch.zeros_like(dh)
    dh[:, 0] = gs * sigma0.clamp(max=E15)
    edh[:, 0] = 2 * U * dh[:, 0].abs()
    s = alb * (1 - alb)
    dh[:, 1:] = dalb * s
    edh[:, 1:] = edalb * s + 4 * U * (dalb * s).abs() + 2 * U * dalb.abs() * alb
    keep = R.in_range.double()[:, None]
    return dh * keep, edh * keep, dtap * keep, edtap * keep, int((amb & R.in_range).sum())


class BwdAcc:
    """fp64 sums of the backward: the table gradient (value, propagated error, magnitude, contribution count) and the weight gradients
    (value, propagated error, magnitude)"""

    def __init__(self, n_entries, dev):
        z = lambda *s: torch.zeros(*s, dtype=torch.float64, device=dev)
        self.table, self.t_err, self.t_mag = z(n_entries, 2), z(n_entries, 2), z(n_entries, 2)
        self.t_cnt = torch.zeros(n_entries, dtype=torch.float64, device=dev)
        shapes = dict(w1=(64, 32), b1=(64,), w2=(64, 64), b2=(64,), w3=(4, 64), b3=(4,))
        self.w = {k: z(*s) for k, s in shapes.items()}
        self.w_err = {k: z(*s) for k, s in shapes.items()}
        self.w_mag = {k: z(*s) for k, s in shapes.items()}
        self.amb_units = 0
        self.units = 0


def backward_eval(f, acc, p, dO, edO):
    """one evaluation point of a chunk: recompute at fp32 positions p, back-propagate dO [n,4] (bound edO), accumulate into acc"""
    m = f.mlp
    u = to_u(p, f.bound)
    enc, e_enc, cs = f.grid.encode(u)
    a = layers(m, enc, e_enc, gamma_bwd)
    z1, e1, h1, z2, e2, h2 = a["z1"], a["e1"], a["h1"], a["z2"], a["e2"], a["h2"]
    live = (dO != 0).any(-1) | (edO != 0).any(-1)
    dH2 = dO @ m.w[2]
    edH2 = edO @ m.a[2] + 5 * U * (dO.abs() @ m.a[2])
    on2, amb2 = z2 > 0, (z2.abs() <= e2) & live[:, None]
    dZ2 = dH2 * on2
    edZ2 = edH2 * (on2 | amb2) + dH2.abs() * amb2
    dH1 = dZ2 @ m.w[1]
    edH1 = edZ2 @ m.a[1] + gamma_bwd(64) * (dZ2.abs() @ m.a[1])
    on1, amb1 = z1 > 0, (z1.abs() <= e1) & live[:, None]
    dZ1 = dH1 * on1
    edZ1 = edH1 * (on1 | amb1) + dH1.abs() * amb1
    dEnc = dZ1 @ m.w[0]
    edEnc = edZ1 @ m.a[0] + gamma_bwd(64) * (dZ1.abs() @ m.a[0])
    acc.amb_units += int(amb1.sum() + amb2.sum())
    acc.units += int(live.sum()) * 128
    h2a, h1a, enca = h2 + e2, h1 + e1, enc.abs() + e_enc

    def add(k, v, err, mag):
        acc.w[k] += v; acc.w_err[k] += err; acc.w_mag[k] += mag
    add("w3", dO.T @ h2, edO.T @ h2a + dO.abs().T @ e2, dO.abs().T @ h2a)
    add("b3", dO.sum(0), edO.sum(0), dO.abs().sum(0))
    add("w2", dZ2.T @ h1, edZ2.T @ h1a + dZ2.abs().T @ e1, dZ2.abs().T @ h1a)
    add("b2", dZ2.sum(0), edZ2.sum(0), dZ2.abs().sum(0))
    add("w1", dZ1.T @ enc, edZ1.T @ enca + dZ1.abs().T @ e_enc, dZ1.abs().T @ enca)
    add("b1", dZ1.sum(0), edZ1.sum(0), dZ1.abs().sum(0))
    for l, (idx, wt) in enumerate(cs):
        g, eg = dEnc[:, 2 * l:2 * l + 2], edEnc[:, 2 * l:2 * l + 2]
        nz = ((g != 0).any(-1) | (eg != 0).any(-1))
        if not bool(nz.any()):
            continue
        idx, wt, g, eg = idx[nz].reshape(-1), wt[nz], g[nz], eg[nz]
        c = (wt[..., None] * g[:, None, :]).reshape(-1, 2)
        ca = c.abs()
        ce = (wt[..., None] * eg[:, None, :]).reshape(-1, 2) + 5 * U * ca
        acc.table.index_add_(0, idx, c)
        acc.t_mag.index_add_(0, idx, ca)
        acc.t_err.index_add_(0, idx, ce)
        acc.t_cnt.index_add_(0, idx, torch.ones_like(idx, dtype=torch.float64))
