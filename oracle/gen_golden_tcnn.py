"""TEST INFRASTRUCTURE ONLY. Runs tiny-cuda-nn's own hash-grid kernels (oracle/_ref/tcnn_grid_ref.so, built by build_ref_tcnn.py from the
reference headers) on a GPU and stores inputs + outputs as tests/golden/tcnn_grid_ref.npz (and tcnn_grid_ref19.npz). Usage:
    python oracle/gen_golden_tcnn.py [OUT.npz]
Configuration: L16 F2, base 32, x2, log2_hashmap_size 16 (level 0 dense, levels 1-15 hashed; 2.03 M parameters -- the table is
regenerated from its seed by the tests, gradients are stored sparsely)."""
import ctypes as C
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
CFG = dict(L=16, log2_hashmap=16, base_res=32, pls=2.0)
SEED, N = 20240923, 256
# round 2: the reference's own geometry (config/base.yaml:10 log2_hashmap_size 19: levels 0-1 dense, 2-15 hashed; 15.27 M parameters),
# a cotangent of the analytic gradient small enough to stay inside the half range at the finest levels, and the input double backward
CFG19 = dict(L=16, log2_hashmap=19, base_res=32, pls=2.0)


def main(out_path, CFG=CFG, cc_scale=1.0):
    lib = C.CDLL(os.path.join(HERE, "_ref", "tcnn_grid_ref.so"))
    lib.tcnn_ref_n_params.restype = C.c_int64
    cfg = (C.c_int(CFG["L"]), C.c_int(CFG["log2_hashmap"]), C.c_int(CFG["base_res"]), C.c_float(CFG["pls"]))
    n_params = lib.tcnn_ref_n_params(*cfg)
    rng = np.random.default_rng(SEED)
    table = rng.uniform(-0.5, 0.5, n_params).astype(np.float32)
    x = rng.uniform(0.0, 1.0, (N, 3)).astype(np.float32)
    x[:8] = rng.choice(np.array([0.0, 1.0, 0.99, 0.985], np.float32), (8, 3))  # cube faces: index wrap of the dense level
    dL_dy = (rng.standard_normal((N, 32)) * 0.05).astype(np.float32)          # cotangent arriving at the encoding's float output
    cc = (rng.standard_normal((N, 3)) * cc_scale).astype(np.float32)          # dL/d(dL/dx)
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    p = lambda tt: C.c_void_p(tt.data_ptr())
    grid_h = t(table).half()                                                   # TCNNModule::forward: params -> half (TB/tcnn_binding.cpp:26-58)
    xt = t(x)
    enc = torch.empty(32, N, dtype=torch.float16, device=dev)
    dy_dx = torch.empty(32 * N * 3, dtype=torch.float32, device=dev)
    assert lib.tcnn_ref_fwd(C.c_int(N), *cfg, p(xt), p(grid_h), p(enc), p(dy_dx)) == 0
    # TCNNModuleFunctionBackward::forward: doutput (half, via the .to(float) backward) * loss_scale, in half (tcnn_binding.cpp:130-134)
    dL_dy_h = (t(dL_dy).half() * 128.0).t().contiguous()                      # SoA [32][N]
    gg = torch.empty(n_params, dtype=torch.float16, device=dev)
    dL_dx = torch.empty(N, 3, dtype=torch.float32, device=dev)
    assert lib.tcnn_ref_bwd(C.c_int(N), *cfg, p(xt), p(dL_dy_h), p(dy_dx), p(gg), p(dL_dx)) == 0
    gg2 = torch.empty(n_params, dtype=torch.float16, device=dev)
    ddy = torch.empty(32, N, dtype=torch.float16, device=dev)
    assert lib.tcnn_ref_bwd_bwd(C.c_int(N), *cfg, p(xt), p(t(cc)), p(dL_dy_h), p(dy_dx), p(gg2), p(ddy)) == 0
    dL_dx2 = torch.empty(N, 3, dtype=torch.float32, device=dev)
    assert lib.tcnn_ref_bwd_bwd_input(C.c_int(N), *cfg, p(xt), p(t(cc)), p(dL_dy_h), p(grid_h), p(dL_dx2)) == 0
    torch.cuda.synchronize()
    sparse = lambda g: (torch.nonzero(g).flatten().cpu().numpy().astype(np.int32), g[torch.nonzero(g).flatten()].float().cpu().numpy())
    i1, v1 = sparse(gg)
    i2, v2 = sparse(gg2)
    os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
    np.savez_compressed(out_path, seed=SEED, n_params=n_params, cfg=np.array([CFG["L"], CFG["log2_hashmap"], CFG["base_res"]]), x=x,
                        dL_dy=dL_dy, cc=cc, enc=enc.t().float().cpu().numpy(), dy_dx=dy_dx.view(32, N, 3).permute(1, 0, 2).cpu().numpy(),
                        dL_dx_scaled=dL_dx.cpu().numpy(), grid_grad_idx=i1, grid_grad_val=v1, grid_grad2_idx=i2, grid_grad2_val=v2,
                        dL_ddLdy=ddy.t().float().cpu().numpy(), dL_dx2_scaled=dL_dx2.cpu().numpy())
    print("wrote", out_path, "nonzeros", len(i1), len(i2))


if __name__ == "__main__":
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "..", "tests", "golden", "tcnn_grid_ref.npz")
    main(out)
    main(out.replace(".npz", "19.npz"), CFG19, cc_scale=1e-3)
