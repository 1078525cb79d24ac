"""
TEST INFRASTRUCTURE (oracle).  Generates tests/golden/ref_py.npz by IMPORTING the reference's own Python helpers
from the exllamav3 checkout of oracle/build_ref.py's reference_root() (the fixture is committed, the reference is not needed by the tests):

  * tensor_core_perm                      modules/quant/exl3_lib/quantize.py:22-44
  * get_hadamard(128) (Sylvester)         util/hadamard.py:107-131
  * preapply_had_l / preapply_had_r       modules/quant/exl3_lib/quantize.py:340-357   on a seeded 256x256 fp16 matrix
  * LinearEXL3.unpack_bf                  modules/quant/exl3.py:142-158                 on a seeded int16 bitfield

The reference package imports its CUDA extension at module import time (exllamav3/ext.py); that import is
stubbed out here because only pure-Python/torch helpers are executed.

usage: python oracle/gen_golden_py.py
"""
import sys, types, os
import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from build_ref import reference_root
REF = reference_root()
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "ref_py.npz")


def import_reference_helpers():
    sys.path.insert(0, REF)
    # stub the compiled extension and heavyweight package __init__s; we only need two leaf modules
    for name in ["exllamav3", "exllamav3.util", "exllamav3.modules", "exllamav3.modules.quant",
                 "exllamav3.modules.quant.exl3_lib", "exllamav3.model", "exllamav3.model.config"]:
        m = types.ModuleType(name)
        m.__path__ = [os.path.join(REF, *name.split("."))]
        sys.modules[name] = m
    ext = types.ModuleType("exllamav3.ext")
    ext.exllamav3_ext = types.SimpleNamespace()
    sys.modules["exllamav3.ext"] = ext
    sys.modules["exllamav3.util"].cuda_sync_active = lambda *a, **k: None
    for stub, attrs in [("exllamav3.util.progress", ["ProgressBar"]),
                        ("exllamav3.util.memory", ["free_mem", "list_gpu_tensors"]),
                        ("exllamav3.util.tensor", ["save_tensor_image", "g_tensor_cache"])]:
        m = types.ModuleType(stub)
        for a in attrs:
            setattr(m, a, type(a, (), {}))
        sys.modules[stub] = m
    sys.modules["exllamav3.model.config"].Config = object
    sys.modules["exllamav3.util"].profile_opt = None
    import importlib
    had = importlib.import_module("exllamav3.util.hadamard")
    q = importlib.import_module("exllamav3.modules.quant.exl3_lib.quantize")
    return had, q


def main():
    had, q = import_reference_helpers()
    out = {}
    out["tensor_core_perm"] = q.tensor_core_perm("cpu").numpy().astype(np.int32)
    out["had128"] = had.get_hadamard(128).float().numpy().astype(np.int8)
    g = torch.Generator().manual_seed(1234)
    w = (torch.randn(256, 256, generator=g) * 1.3).half()
    out["had_in"] = w.numpy()
    out["had_l"] = q.preapply_had_l(w, 128).numpy()
    out["had_r"] = q.preapply_had_r(w, 128).numpy()
    # unpack_bf is a method that does not touch self except transformers_fix
    src = open(os.path.join(REF, "exllamav3/modules/quant/exl3.py")).read()
    bits = torch.randint(-32768, 32767, (16,), generator=g, dtype=torch.int16)
    ns = {}
    import textwrap, re
    body = src[src.index("    def unpack_bf"):src.index("    def reconstruct_hgemm")]
    exec("import torch\n" + textwrap.dedent(body), ns)
    out["bf_in"] = bits.numpy()
    out["bf_out"] = ns["unpack_bf"](types.SimpleNamespace(transformers_fix=False), bits).numpy()
    np.savez_compressed(OUT, **out)
    print("wrote", os.path.abspath(OUT), {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
