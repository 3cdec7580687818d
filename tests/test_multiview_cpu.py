"""Host-only planning of the SD engine for G views (mi3d_sd_workspace_bytes needs no GPU): U-Net batch 2G and VAE encoder batch G plan
for every G up to MI3D_MAX_VIEWS, and the GroupNorm-statistics pool grows with the batch instead of refusing it."""
import ctypes as C
import importlib

sdm = importlib.import_module("make-it-3d_b200.nerf.sd")
L = importlib.import_module("make-it-3d_b200._lib")


def _bytes(unet=None, vae=None):
    lib = L.lib()
    lib.mi3d_sd_workspace_bytes.restype = C.c_size_t
    return lib.mi3d_sd_workspace_bytes(C.byref(unet) if unet is not None else None, C.byref(vae) if vae is not None else None)


def test_g_view_engines_plan_at_full_size():
    ucfg, vcfg = sdm.sd20_unet_cfg(), dict(sdm.sd_vae_cfg(), decoder=False)
    unet = [_bytes(unet=sdm._unet_struct(ucfg, G)) for G in range(1, L.MAX_VIEWS + 1)]
    vae = [_bytes(vae=sdm._vae_struct(vcfg, G)) for G in range(1, L.MAX_VIEWS + 1)]
    assert all(b > 0 for b in unet + vae), (unet, vae)          # batch 16 used to overflow the fixed 256 KB statistics pool
    assert all(a < b for a, b in zip(unet, unet[1:])) and all(a < b for a, b in zip(vae, vae[1:]))
    # the encoder tape is per image: G images take about G times one image's
    assert 0.9 * L.MAX_VIEWS < vae[-1] / vae[0] < 1.1 * L.MAX_VIEWS
    # mi3d_vae_cfg.batch 0 and 1 both mean one image
    zero = sdm._vae_struct(vcfg, 1)
    zero.batch = 0
    assert _bytes(vae=zero) == vae[0]
    neg = sdm._vae_struct(vcfg, 1)
    neg.batch = -1
    assert _bytes(vae=neg) == 0
