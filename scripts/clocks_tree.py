"""Phase clocks of the fused step kernel for any checked-out tree: python scripts/clocks_tree.py TREE B [split_from]
(steady state: 14 warm-up steps so that older trees have primed every stream)."""
import os, sys
tree = os.path.abspath(sys.argv[1]); os.chdir(tree); sys.path.insert(0, tree)
import numpy as np
from openwakeword_b200.engine import StreamEngine
from openwakeword_b200 import weights as W
B = int(sys.argv[2]); split = int(sys.argv[3]) if len(sys.argv) > 3 else None
kw = dict(cnn_mode=3)
if split is not None: kw["split_from"] = split
eng = StreamEngine([W.synthetic_head(seed=1)], B, **kw)
rng = np.random.default_rng(0)
for _ in range(14):
    eng.step_host(rng.integers(-1000, 1000, (B, 1280)).astype(np.int16), 1)
NL = split if split is not None and split < 20 else 20
for rep in range(2):
    eng.ctx.debug_inc_clocks_arm()
    eng.step_host(rng.integers(-1000, 1000, (B, 1280)).astype(np.int16), 1)
    c = eng.ctx.debug_inc_clocks_read()
    st = list(c[:NL]) + [c[20]]
    print(f"{os.path.basename(tree)} B={B} split={split}: phase cyc:", np.diff(st).tolist(), " layers total", int(c[20] - c[0]), "cyc")
    print("  first accumulator:", c[61:61 + NL].tolist())
    print("  to last store:", c[81:81 + NL].tolist())
    print("  frontend:", int(c[0] - c[101]), " heads:", int(c[102] - c[20]) if c[102] else None)
    if c[92]:
        print("  frontend detail (warp 0, first frame pair): start +%d | load+window %d | FFT %d | unpack %d | mel+log %d ; all frames done +%d ; floor/affine/ring/tail %d" % (
            c[92] - c[101], c[93] - c[92], c[94] - c[93], c[95] - c[94], c[96] - c[95], c[97] - c[101], c[0] - c[97]))
