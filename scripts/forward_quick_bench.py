"""Quick device-side timing of the pairwise forward + the main GEMM shapes (iteration aid)."""
import sys, os, json, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from dust3r_b200 import _lib
from dust3r_b200.config import vitl_512_dpt
from dust3r_b200.model import AsymmetricCroCo3DStereo
from dust3r_b200.utils.synth import synth_state_dict

def timeit(fn, warm=2, rep=5):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(rep): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / rep

def gemm_shapes():
    lib = _lib.get_lib()
    dev = 'cuda'
    for (M, N, K, fl) in [(49152, 3072, 1024, 1), (49152, 1024, 1024, 1), (49152, 4096, 1024, 3), (49152, 1024, 4096, 1 | 16),
                          (24576, 2304, 768, 1), (24576, 768, 768, 1), (24576, 3072, 768, 3), (24576, 768, 3072, 1 | 16)]:
        A = torch.randn((M, K), device=dev).bfloat16(); B = torch.randn((N, K), device=dev).bfloat16()
        bias = torch.randn((N,), device=dev)
        out = torch.zeros((M, N), device=dev, dtype=torch.float32 if fl & 16 else torch.bfloat16)
        def f():
            _lib.check(lib.d3r_gemm_bf16(A.data_ptr(), B.data_ptr(), out.data_ptr(), bias.data_ptr(), None, None, M, N, K, N, fl, None, None, 0, 0, 0, _lib.stream_ptr()))
        ms = timeit(f)
        ref = timeit(lambda: torch.matmul(A, B.T))
        print(json.dumps(dict(kind='gemm', M=M, N=N, K=K, flags=fl, ms=ms, tflops=2 * M * N * K / ms / 1e9, cublas_ms=ref, cublas_tflops=2 * M * N * K / ref / 1e9)), flush=True)

def forward(Bp):
    cfg = vitl_512_dpt()
    net = AsymmetricCroCo3DStereo(pos_embed='RoPE100', img_size=(512, 512), head_type='dpt', enc_embed_dim=1024, enc_depth=24,
                                  enc_num_heads=16, dec_embed_dim=768, dec_depth=12, dec_num_heads=12, landscape_only=False)
    net.load_state_dict(synth_state_dict(cfg, 0)); net = net.to('cuda')
    packed = net.repack()
    H, W = 384, 512
    for B in Bp:
        imgs = (torch.rand((2 * B, 3, H, W), device='cuda') * 2 - 1)
        idx1, idx2 = np.arange(B, dtype=np.int32), B + np.arange(B, dtype=np.int32)
        ms = timeit(lambda: packed.forward(imgs, idx1, idx2, B, H, W), warm=2, rep=3)
        print(json.dumps(dict(kind='forward', B=B, ms=ms, pairs_per_s=B / ms * 1e3, tflops_alg=B * 1856.8 / ms)), flush=True)
        packed._ws.clear()

if __name__ == '__main__':
    lib = _lib.get_lib()
    for impl in (2, 1):
        lib.d3r_set_gemm_impl(impl)
        print(json.dumps(dict(kind='gemm_impl', impl=impl)), flush=True)
        gemm_shapes()
        forward([8, 32])
