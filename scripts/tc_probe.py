"""Small driver for ncu: K2 (wgmma) dense search, batch 256, over a device-generated corpus."""
import sys
import numpy as np
sys.path.insert(0, ".")
from kaito_b200 import _native

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
batch = int(sys.argv[2]) if len(sys.argv) > 2 else 256
mode = int(sys.argv[3]) if len(sys.argv) > 3 else _native.DENSE_TC
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 3
ctx = _native.Context(0, dense_mode=mode)
ix = ctx.create_index("probe", 768)
ix.synth_fill(n, 0, 5)
g = np.random.default_rng(0)
q = g.standard_normal((batch, 768)).astype(np.float32)
q /= np.linalg.norm(q, axis=1, keepdims=True)
for _ in range(reps):
    d, o = ix.search_dense(q, 30)
print("ok", d[0, :3], o[0, :3], "fallbacks", _native.load().krag_tc_fallback_queries())
ix.drop(); ctx.close()
