"""Generate tests/golden/vqgan_reference_small.npz by EXECUTING THE REFERENCE MODULE lwm/vqgan.py of a
LargeWorldModel/LWM checkout (its root is $LWM_REFERENCE; unmodified) over the numpy-backed flax/jax shim in oracle/flax_shim (see its README for what this does and does not
pin). The fixture is committed, so the tests need no reference checkout.

Config: a down-scaled VQGANConfig (resolution 64, hidden 32, codebook 512) so that the fixture stays small; layer
structure, naming and every code path of encode()/decode() are those of the default config."""
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "flax_shim"))
sys.path.insert(1, ROOT)

CFG = dict(resolution=64, hidden_channels=32, num_embeddings=512)


def to_np_tree(t):
    return {k: (to_np_tree(v) if isinstance(v, dict) else np.asarray(v, dtype=np.float32)) for k, v in t.items()}


def main():
    spec = importlib.util.spec_from_file_location(
        "lwm_ref_vqgan", os.path.join(os.environ.get("LWM_REFERENCE", "reference"), "lwm", "vqgan.py"))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)
    from oracle import vqgan_ref as vr

    params = vr.init_params(CFG, seed=3, codebook="normal")
    np_params = to_np_tree(params)
    config = ref.VQGANConfig.get_default_config(CFG)
    model = ref.VQGANModel(config)
    g = torch.Generator().manual_seed(5)
    pixels = (torch.rand(2, 64, 64, 3, generator=g) * 2 - 1).numpy().astype(np.float32)
    video = pixels.reshape(1, 2, 64, 64, 3)
    zq, idx = model.apply({"params": np_params}, video, method=model.encode)          # [B,T,...] branch
    codes = np.random.default_rng(7).integers(0, 512, size=(2, 4, 4))
    recon = model.apply({"params": np_params}, codes, method=model.decode)
    out = os.path.join(ROOT, "tests", "golden", "vqgan_reference_small.npz")
    np.savez_compressed(out, pixels=pixels, zq=np.asarray(zq, np.float32), idx=np.asarray(idx).astype(np.int32),
                        codes=codes.astype(np.int32), recon=np.asarray(recon, np.float32),
                        cfg_resolution=64, cfg_hidden=32, cfg_codes=512, param_seed=3)
    print("wrote", out, "zq", zq.shape, "idx", idx.shape, "recon", recon.shape)


if __name__ == "__main__":
    main()
