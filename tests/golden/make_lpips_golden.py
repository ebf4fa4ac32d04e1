"""Golden LPIPS values from the reference's OWN lpipsPyTorch (gaussian_splatting/lpipsPyTorch).

Runs where the reference sources are present:  python tests/golden/make_lpips_golden.py
Imports the package from /root/reference by path and runs its `LPIPS('vgg', '0.1')` unchanged, with two stubs in
place of the downloads: torchvision.models.vgg16 returns vgg16(weights=None) loaded with the seeded weights of
tests/lpips_cases.py, and torch.hub.load_state_dict_from_url returns the seeded linear layers.  Nothing of the
reference is copied; only the numbers are stored.
Output: tests/golden/lpips_values.npz, holding the weights' seed and digest (the ~59 MB of weights are regenerated,
not stored), and per case <name>_x, <name>_y (float32 inputs), <name>_lpips_f32/_f64 (the module's output: for
N > 1 the reference's sum over the batch) and <name>_taps_f32/_f64 ([N, 5]: each tap's per-image mean, computed by
the module's own net and lin layers as its forward does).
"""
import importlib.util
import io
import os
import sys
import zipfile

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import lpips_cases as lc  # noqa: E402

REF = "/root/reference/gaussian_splatting/lpipsPyTorch"


def import_reference(vgg_sd, lin_sd):
    plain_vgg16 = torchvision.models.vgg16

    def vgg16(weights=None, **_):
        m = plain_vgg16(weights=None)
        m.load_state_dict({**m.state_dict(), **vgg_sd})
        return m

    def load_state_dict_from_url(url, **_):
        assert url.endswith("/v0.1/vgg.pth"), url
        return dict(lin_sd)

    torchvision.models.vgg16 = vgg16
    torch.hub.load_state_dict_from_url = load_state_dict_from_url
    spec = importlib.util.spec_from_file_location("ref_lpipsPyTorch", os.path.join(REF, "__init__.py"),
                                                  submodule_search_locations=[REF])
    mod = importlib.util.module_from_spec(spec)
    sys.modules["ref_lpipsPyTorch"] = mod
    spec.loader.exec_module(mod)
    return mod


def run(mod, x, y, dtype):
    crit = mod.modules.lpips.LPIPS("vgg", "0.1").to(dtype).eval()
    x, y = x.to(dtype), y.to(dtype)
    with torch.no_grad():
        total = crit(x, y).reshape(-1)
        fx, fy = crit.net(x), crit.net(y)
        taps = torch.stack([l((a - b) ** 2).mean((1, 2, 3)) for a, b, l in zip(fx, fy, crit.lin)], 1)
    return total.numpy(), taps.numpy()


def save_deterministic(path, arrays):
    """np.savez with fixed zip timestamps so that the file's bytes depend on its arrays only."""
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, buf.getvalue())


def main():
    torch.set_num_threads(1)
    vgg_sd, lin_sd = lc.make_state_dicts(lc.WEIGHT_SEED)
    mod = import_reference(vgg_sd, lin_sd)
    out = {"weight_seed": np.int64(lc.WEIGHT_SEED),
           "weight_digest": np.frombuffer(bytes.fromhex(lc.digest(vgg_sd, lin_sd)), np.uint8)}
    for name, N, H, W, noise, seed in lc.GOLDEN_CASES:
        x, y = lc.image_pair(N, H, W, noise, seed)
        out[name + "_x"], out[name + "_y"] = x.numpy(), y.numpy()
        for dt, tag in ((torch.float32, "f32"), (torch.float64, "f64")):
            out[f"{name}_lpips_{tag}"], out[f"{name}_taps_{tag}"] = run(mod, x, y, dt)
        print(name, out[f"{name}_lpips_f64"], out[f"{name}_taps_f64"].sum(1))
    path = os.path.join(HERE, "lpips_values.npz")
    save_deterministic(path, out)
    print(path, os.path.getsize(path))


if __name__ == "__main__":
    main()
