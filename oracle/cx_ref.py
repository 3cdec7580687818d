"""fp32 / fp64 PyTorch restatement of the contextual loss the refine stage uses (nerf/utils.py:36, 455-457, 810, 882):
`contextual_loss.ContextualLoss(band_width=0.5, loss_type='cosine', use_vgg=True, vgg_layer='relu5_4')` of the pip package
S-aiueo32/contextual_loss_pytorch.  The package is not installed; this restates its published source:

1. x' = (x - mean) / std with ImageNet mean (0.485, 0.456, 0.406) and std (0.229, 0.224, 0.225); the same for y.
2. features = torchvision vgg19().features[0:36] (conv1_1 .. relu5_4, no pool5), frozen, held by the package's VGG19 in five
   slices: slice1 = features[0:4], slice2 = [4:9], slice3 = [9:18], slice4 = [18:27], slice5 = [27:36]; so the state_dict names are
   vgg_model.slice{s}.{index}.{weight,bias}.  MaxPool2d(2, 2) floors odd sizes.
3. y_mu = y_feat.mean(dim=(0, 2, 3)) (over the batch too); both maps are centred by y_mu, then F.normalize(dim=1, eps=1e-12).
4. d[n, i, j] = 1 - <x_i, y_j> over positions i of x and j of y.
5. d~ = d / (min_j d + 1e-5).
6. w = exp((1 - d~) / band_width); cx = w / sum_j w.
7. loss = mean_n(-log(mean_j max_i cx[n, i, j] + 1e-5)).

The gradient flows to x only.  Ties in min / max go to the lowest index (torch's rule); max-pool ties to the first element in
row-major window order.
"""
import torch
import torch.nn.functional as F

MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
# torchvision vgg19().features[0:36]: conv (index, out channels) and pools
LAYERS = [("conv", 0, 64), ("conv", 2, 64), ("pool", 4, 0), ("conv", 5, 128), ("conv", 7, 128), ("pool", 9, 0),
          ("conv", 10, 256), ("conv", 12, 256), ("conv", 14, 256), ("conv", 16, 256), ("pool", 18, 0),
          ("conv", 19, 512), ("conv", 21, 512), ("conv", 23, 512), ("conv", 25, 512), ("pool", 27, 0),
          ("conv", 28, 512), ("conv", 30, 512), ("conv", 32, 512), ("conv", 34, 512)]


def slice_of(idx):
    return 1 if idx < 4 else 2 if idx < 9 else 3 if idx < 18 else 4 if idx < 27 else 5


def package_to_torchvision():
    """{'vgg_model.sliceS.N.weight': 'features.N.weight', ...} for every tensor of the 16 convs"""
    out = {}
    for kind, idx, _ in LAYERS:
        if kind == "conv":
            for leaf in ("weight", "bias"):
                out[f"vgg_model.slice{slice_of(idx)}.{idx}.{leaf}"] = f"features.{idx}.{leaf}"
    return out


def normalize_images(x):
    m = torch.tensor(MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    s = torch.tensor(STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - m) / s


def vgg_features(x, params, round_fp16=False):
    """features[0:36] of x (already normalised); params: package names -> tensors.  round_fp16: round every layer output to fp16
    (the storage the engine uses), for the tests' precision floor."""
    h = x
    for kind, idx, _ in LAYERS:
        if kind == "pool":
            h = F.max_pool2d(h, 2, 2)
        else:
            pre = f"vgg_model.slice{slice_of(idx)}.{idx}"
            h = F.relu(F.conv2d(h, params[pre + ".weight"].to(h.dtype), params[pre + ".bias"].to(h.dtype), padding=1))
        if round_fp16:
            h = h.half().to(x.dtype)
    return h


def cx_from_features(xf, yf, band_width=0.5):
    """steps 3-7, vectorised as the package's functional.contextual_loss"""
    y_mu = yf.mean(dim=(0, 2, 3), keepdim=True)
    xn = F.normalize(xf - y_mu, p=2, dim=1)
    yn = F.normalize(yf - y_mu, p=2, dim=1)
    N, Cc = xf.shape[:2]
    xn = xn.reshape(N, Cc, -1)
    yn = yn.reshape(N, Cc, -1)
    dist = 1 - torch.bmm(xn.transpose(1, 2), yn)
    dist_min, _ = torch.min(dist, dim=2, keepdim=True)
    dist_tilde = dist / (dist_min + 1e-5)
    w = torch.exp((1 - dist_tilde) / band_width)
    cx = w / torch.sum(w, dim=2, keepdim=True)
    cx = torch.mean(torch.max(cx, dim=1)[0], dim=1)
    return torch.mean(-torch.log(cx + 1e-5))


def cx_from_features_loop(xf, yf, band_width=0.5):
    """steps 3-7 in explicit loops (float64), an independent restatement of cx_from_features"""
    xf, yf = xf.double(), yf.double()
    N, Cc, H, W = xf.shape
    P = H * W
    y_mu = [sum(float(yf[n, c].sum()) for n in range(N)) / (N * P) for c in range(Cc)]
    mu = torch.tensor(y_mu, dtype=torch.float64).view(1, Cc, 1, 1)
    total = 0.0
    for n in range(N):
        xr = (xf[n] - mu[0]).reshape(Cc, P).T
        yr = (yf[n] - mu[0]).reshape(Cc, P).T
        xr = [r / max(float(r.norm()), 1e-12) for r in xr]
        yr = [r / max(float(r.norm()), 1e-12) for r in yr]
        cx = [[0.0] * P for _ in range(P)]
        for i in range(P):
            d = [1.0 - float(xr[i] @ yr[j]) for j in range(P)]
            dmin = min(d)
            w = [torch.exp(torch.tensor((1.0 - dj / (dmin + 1e-5)) / band_width, dtype=torch.float64)).item() for dj in d]
            s = sum(w)
            cx[i] = [wj / s for wj in w]
        m = sum(max(cx[i][j] for i in range(P)) for j in range(P)) / P
        total += -torch.log(torch.tensor(m + 1e-5, dtype=torch.float64)).item()
    return total / N


def contextual_loss(x, y, params, band_width=0.5, round_fp16=False):
    """the full loss: x, y [N,3,H,W] in [0, 1]-ish image space"""
    xf = vgg_features(normalize_images(x), params, round_fp16)
    yf = vgg_features(normalize_images(y), params, round_fp16)
    return cx_from_features(xf, yf, band_width)


def seeded_params(seed=0, device="cpu"):
    """seeded VGG19 weights under the package's names (kaiming-normal fan_in weights, non-zero biases)"""
    g = torch.Generator().manual_seed(seed)
    out, cin = {}, 3
    for kind, idx, cout in LAYERS:
        if kind != "conv":
            continue
        pre = f"vgg_model.slice{slice_of(idx)}.{idx}"
        out[pre + ".weight"] = (torch.randn(cout, cin, 3, 3, generator=g) * (2.0 / (cin * 9)) ** 0.5).to(device)
        out[pre + ".bias"] = (torch.randn(cout, generator=g) * 0.05).to(device)
        cin = cout
    return out
