"""Quick device-resident timing of the DTD GEMM window (development aid, not the bench)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from parsec_b200 import _lib as L
from oracle import orc_dags as dags
from parsec_b200.engine import Engine

NT = int(sys.argv[1]) if len(sys.argv) > 1 else 16
T = int(sys.argv[2]) if len(sys.argv) > 2 else 512
modes = [int(x) for x in sys.argv[3].split(",")] if len(sys.argv) > 3 else [0, 2]
tb = T * T * 2
for mode in modes:
    with Engine(0, gemm_mode=mode) as e:
        dag = dags.dtd_gemm(NT, T)
        dag.tasks["access"][:, 2] &= ~np.uint8(L.FLOW_PUSHOUT)
        slab = e.malloc(dag.ntiles * tb)
        init = np.full(dag.ntiles * tb // 2, 0x3C00, np.uint16)
        e.h2d(slab, init)
        tiles = np.zeros(dag.ntiles, L.TILE_DTYPE)
        tiles["dev_ptr"] = slab + np.arange(dag.ntiles, dtype=np.uint64) * np.uint64(tb)
        tiles["bytes"] = tb
        tiles["state"] = L.TILE_VALID
        w = e.window(1, dag.tasks, dag.succ, tiles, dag.ready)
        flops = 2.0 * (NT * T) ** 3
        for it in range(3):
            st = w.run()
        ms = min(w.run()["kernel_ms"] for _ in range(3))
        print(f"mode={mode} NT={NT} T={T} kernel_ms={ms:.3f} tasks/s={dag.ntasks/ms*1e3:.3e} TFLOP/s={flops/ms/1e9:.1f}")
        w.close()
