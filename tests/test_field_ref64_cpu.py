"""CPU pin of tests/field_ref64.py (the fp64 restatement the field parity tests compare the kernels with) against oracle/field_ref.FieldRef
plus autograd, which tests/test_oracle_golden.py holds to the vectors recorded from the reference's own Python.  About 2 k samples,
every shading, n_evals 1 / 7 / 13, the two loss terms with an injected smoothing perturbation, and the backward of all of it.

FieldRef runs with float64 parameters on the same fp32 positions (its position arithmetic follows the dtype of x), so the two
restatements differ only by the fp32 corner weights of HashGridRef and its fp32 blob, which the normals amplify by 1 / (2 eps) = 50: 1e-5 relative (1e-4 for the gradients) covers that.  (In fp32, autograd's
own rounding of the +-0.01 tap gradients, which cancel in dW1, reaches 1e-2 of the largest entry.)"""
import numpy as np
import pytest
import torch

import field_ref64 as F
from helpers import fr, make_table

M = 2048
TWO_R2 = float(torch.tensor(2.0 * float(torch.tensor(0.1, dtype=torch.float32)) ** 2, dtype=torch.float32))


def _setup(seed=0):
    f = fr.FieldRef(bound=1.0, blob_density=5.0, blob_radius=0.1, seed=seed)
    table = make_table(f.encoder.params.numel(), 7, 0.5)
    with torch.no_grad():
        f.encoder.params.copy_(torch.from_numpy(table))
    f = f.double()
    f.gaussian = lambda x: f.blob_density * torch.exp(-(x.double() ** 2).sum(-1) / TWO_R2)     # fp64 blob on the fp32 positions
    lv = f.encoder.levels
    L = f.encoder.n_levels
    grid = F.Grid(lv["offsets"][:L], lv["sizes"][:L], lv["ress"][:L], lv["scales"][:L], torch.from_numpy(table))
    net = f.sigma_net.net
    mlp = F.Mlp(*(t.detach() for t in (net[0].weight, net[0].bias, net[1].weight, net[1].bias, net[2].weight, net[2].bias)))
    rng = np.random.default_rng(seed + 1)
    x = ((rng.random((M, 3), dtype=np.float32) * 2 - 1) * 0.6).astype(np.float32)
    x[:3] = np.array([[1, 1, 1], [-1, 0.5, 0.2], [0.995, 0, 0]], np.float32)        # faces and a tap that leaves the box
    d = rng.standard_normal((M, 3)).astype(np.float32); d /= np.linalg.norm(d, axis=1, keepdims=True)
    z = rng.standard_normal((M, 3)).astype(np.float32)
    l = np.array([0.3, 0.5, 0.81], np.float32); l /= np.linalg.norm(l)
    return f, F.Field64(grid, mlp), torch.from_numpy(x), torch.from_numpy(d), torch.from_numpy(z), torch.from_numpy(l)


def _rows(x, d, z, l):
    n = x.shape[0]
    ones = torch.ones(n, dtype=torch.bool)
    return F.Rows(x, d, F.perturbed(x, z), ones, ones, torch.zeros(n, dtype=torch.long), torch.full((n,), n, dtype=torch.long),
                  l.double().expand(n, 3))


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / max(1e-12, float(b.abs().max())))


@pytest.mark.parametrize("shading,ratio", [("albedo", 1.0), ("lambertian", 0.1), ("textureless", 0.2), ("normal", 0.1)])
@pytest.mark.parametrize("n_evals", [1, 7, 13])
def test_field_ref64_matches_oracle_field_ref(shading, ratio, n_evals):
    if n_evals == 1 and shading != "albedo":
        pytest.skip("one evaluation has no normal: only albedo is meaningful")
    f, f64, x, d, z, l = _setup()
    R = _rows(x, d, z, l)
    out = f64.forward(R, n_evals, shading, ratio)
    # rows with a hidden unit within 1e-6 of its ReLU kink take no gradient: HashGridRef's fp32 corner weights can flip such a unit
    far = torch.ones(M, dtype=torch.bool)
    for e in range(n_evals):
        a = f64.eval_point(F.eval_pos(e, R.x, R.xp, f64.bound))["layers"]
        far &= (a["z1"].abs().min(-1).values > 1e-6) & (a["z2"].abs().min(-1).values > 1e-6)
    assert int(far.sum()) > 0.95 * M
    w = far.double()
    gs = torch.randn(M, generator=torch.Generator().manual_seed(1)).double() * w
    gc = torch.randn(M, 3, generator=torch.Generator().manual_seed(2)).double() * w[:, None]
    gn = torch.randn(M, 3, generator=torch.Generator().manual_seed(3)).double() * 0.1 * w[:, None]
    Go, Gs = 0.7, 0.3
    if n_evals == 1:
        ref = f.density(x)
        sig_r, col_r = ref["sigma"], ref["albedo"]
        loss = (sig_r * gs).sum() + (col_r * gc).sum()
    else:
        sig_r, col_r, nrm_r = f(x, d, l.double(), ratio=ratio, shading=shading)
        assert _rel(out["normal"], nrm_r.detach()) < 1e-5
        weights = 1 - torch.exp(-sig_r)
        to = weights.detach() * (nrm_r * d).sum(-1).clamp(min=0) ** 2
        assert abs(float(out["t_orient"].mean()) / float(to.mean()) - 1) < 1e-5
        loss = (sig_r * gs).sum() + (col_r * gc).sum() + (nrm_r * gn).sum() + Go * (to * w).mean()
        if n_evals == 13:
            ts = (nrm_r - f.normal(R.xp)).abs()
            assert abs(float(out["t_smooth"].sum()) / (3 * M) / float(ts.mean()) - 1) < 1e-5
            loss = loss + Gs * (ts * w[:, None]).mean()
    assert _rel(out["sigma"], sig_r.detach()) < 1e-6
    assert (out["rgb"] - col_r.detach().double()).abs().max() < 1e-5
    loss.backward()
    # the fp64 backward from the fp64 tape
    acc = F.BwdAcc(f64.grid.table.shape[0], "cpu")
    Gov = w * Go / M if n_evals >= 7 else torch.zeros(M, dtype=torch.float64)
    Gsv = w * Gs / (3 * M) if n_evals == 13 else torch.zeros(M, dtype=torch.float64)
    dh, _, dtap, _, _ = F.out_grads(out["tape"], R, gs, gc, gn if n_evals >= 7 else torch.zeros(M, 3), Gov, Gsv, n_evals,
                                    shading, ratio, n_evals == 13)
    for e in range(n_evals):
        dO = dh if e == 0 else torch.nn.functional.pad(dtap[:, e - 1:e], (0, 3))
        F.backward_eval(f64, acc, F.eval_pos(e, R.x, R.xp, f64.bound), dO, torch.zeros_like(dO))
    net = f.sigma_net.net
    for k, p in (("w1", net[0].weight), ("b1", net[0].bias), ("w2", net[1].weight), ("b2", net[1].bias), ("w3", net[2].weight),
                 ("b3", net[2].bias)):
        assert _rel(acc.w[k], p.grad) < 1e-4, k
    gt = f.encoder.params.grad.view(-1, 2)
    assert _rel(acc.table, gt) < 1e-4
    assert not bool(((gt != 0).any(-1) & (acc.t_cnt == 0)).any())      # every entry autograd touches has a counted contribution


def test_philox_restatement_known_values():
    """Philox4x32-10 test vectors of Salmon et al. (Random123 kat_vectors): counter / key all zero and all ones"""
    z = torch.zeros(1, dtype=torch.long)
    r = F.philox((z, z, z, z), (0, 0))
    assert [int(v) for v in r] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    o = z + 0xFFFFFFFF
    r = F.philox((o, o, o, o), (0xFFFFFFFF, 0xFFFFFFFF))
    assert [int(v) for v in r] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]
