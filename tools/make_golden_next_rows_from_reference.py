"""Generate tests/golden/rope_reference.npz and tests/golden/vision_tokens_reference.npz by EXECUTING REFERENCE CODE
(unmodified source text, extracted with `ast` from a checkout of LargeWorldModel/LWM at run time — nothing is copied
into this repo; the checkout's root is $LWM_REFERENCE):
  * lwm/llama.py `precompute_freqs_cis` and `apply_rotary_emb` over the numpy-backed jax shim (oracle/flax_shim);
  * lwm/data.py `VisionTextProcessor` with a stub tokenizer (only `<vision>` / `</vision>` / bos / eos ids matter).
The fixtures are committed, so the tests need no reference checkout."""
import ast
import os
import random
import sys
from typing import Tuple  # noqa: F401  (names the extracted source refers to)

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle", "flax_shim"))
REF = os.path.join(os.environ.get("LWM_REFERENCE", "reference"), "lwm")


def extract(path, names):
    src = open(path).read()
    tree = ast.parse(src)
    out = []
    for node in tree.body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)) and node.name in names:
            out.append(ast.get_source_segment(src, node))
    assert len(out) == len(names), (path, names)
    return "\n\n".join(out)


def make_rope():
    import jax
    import jax.numpy as jnp
    ns = dict(np=np, jnp=jnp, jax=jax, Tuple=Tuple)
    exec(extract(os.path.join(REF, "llama.py"), ["precompute_freqs_cis", "apply_rotary_emb"]), ns)
    rng = np.random.default_rng(11)
    B, S, H, D = 2, 48, 3, 128
    out = {}
    for tag, theta, max_pos in (("t1e4", 10000.0, 4096), ("t5e7", 50000000.0, 1048576)):
        table = np.asarray(ns["precompute_freqs_cis"](D, max_pos, theta=theta))
        # positions: a contiguous run, a far-out run (needs accurate range reduction) and scattered ones
        pos = np.stack([np.arange(S), np.concatenate([np.arange(max_pos - S // 2, max_pos),
                                                      rng.integers(0, max_pos, S - S // 2)])]).astype(np.int32)
        xq = rng.standard_normal((B, S, H, D)).astype(np.float32)
        xk = rng.standard_normal((B, S, 2, D)).astype(np.float32)
        freqs = np.take(table, pos, axis=0)                                   # llama.py:515
        oq, ok = ns["apply_rotary_emb"](xq, xk, freqs_cis=freqs, dtype=np.float32)
        out.update({tag + "_pos": pos, tag + "_xq": xq, tag + "_xk": xk, tag + "_oq": np.asarray(oq, np.float32),
                    tag + "_ok": np.asarray(ok, np.float32), tag + "_theta": theta, tag + "_max_pos": max_pos,
                    tag + "_cos": table.real[pos].astype(np.float32), tag + "_sin": table.imag[pos].astype(np.float32)})
    path = os.path.join(ROOT, "tests", "golden", "rope_reference.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: getattr(v, "shape", v) for k, v in out.items()})


class StubTokenizer:
    bos_token_id, eos_token_id = 1, 2

    def encode(self, text):
        return {"<vision>": [32000], "</vision>": [32001, 32002]}.get(text, [100 + (ord(c) % 50) for c in text])


def make_vision_tokens():
    from ml_collections import ConfigDict
    ns = dict(np=np, random=random, ConfigDict=ConfigDict)
    exec(extract(os.path.join(REF, "data.py"), ["VisionTextProcessor"]), ns)
    rng = np.random.default_rng(13)
    out = {}
    for tag, n_frames, max_n in (("f1", 1, -1), ("f5", 5, -1), ("f9sel4", 9, 4)):
        proc = ns["VisionTextProcessor"](dict(fields_from_example="fields", max_n_frames=max_n), StubTokenizer())
        codes = rng.integers(0, 8192, size=n_frames * 256)
        example = {"fields": "vision", "vision": codes.tolist()}
        tokens, loss_mask, vmask, keep, *_ = proc((example, 0), has_aux=True)
        out.update({tag + "_codes": codes.astype(np.int32), tag + "_tokens": np.asarray(tokens, np.int32),
                    tag + "_vision_mask": np.asarray(vmask, bool), tag + "_max_n_frames": max_n})
    path = os.path.join(ROOT, "tests", "golden", "vision_tokens_reference.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, {k: getattr(v, "shape", v) for k, v in out.items()})


if __name__ == "__main__":
    make_rope()
    make_vision_tokens()


def make_process_frame_fixture(path="tests/golden/process_frame_reference.npz"):
    """tests/golden/process_frame_reference.npz: outputs of the reference's own `Sampler._process_frame`
    (lwm/vision_chat.py:59-74), source text extracted with ast and executed, on the seeded images of
    tests/test_next_rows2_cpu.py::_images at size 64."""
    import ast
    import sys
    import numpy as np
    sys.path.insert(0, "tests")
    from test_next_rows2_cpu import _images
    src = open(os.path.join(REF, "vision_chat.py")).read()
    fn = next(n for n in ast.walk(ast.parse(src)) if isinstance(n, ast.FunctionDef) and n.name == "_process_frame")
    ns = {"np": np}
    exec("def _process_frame" + ast.get_source_segment(src, fn).split("def _process_frame", 1)[1], ns)
    np.savez_compressed(path, **{"frame_%d" % i: ns["_process_frame"](None, im, 64) for i, im in enumerate(_images())})
