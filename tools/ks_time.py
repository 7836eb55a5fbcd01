"""Key-switch time by batch (CUDA events, 5 calls after 2 warm-up calls) for a random key whose d = 0 rows are zero, as
in every generated key.  With a build that has nb_ks_prepare the key is prepared first, so batches from the library's
threshold up run the tensor-core GEMM.  Run from the repository root."""
import sys, torch
sys.path.insert(0, '.')
from nufhe_b200.engine import Engine
eng = Engine(0)
g = torch.Generator().manual_seed(1)
def r(shape): return torch.randint(-2**31, 2**31, shape, generator=g, dtype=torch.int64).to(torch.int32).cuda()
ks = (r((1024,8,4,500)), r((1024,8,4)), torch.zeros((1024,8,4), dtype=torch.float32).cuda())
ks[0][:, :, 0] = 0
ks[1][:, :, 0] = 0
planes = eng.ks_prepare(ks[0], ks[1]) if hasattr(eng, 'ks_prepare') else None
print('prepared' if planes is not None else 'not prepared')
for B in (1, 16, 64, 148, 256, 592, 1024, 2048, 2368, 4096, 8192, 16384):
    src = (r((B,1024)), r((B,)))
    for _ in range(2): eng.keyswitch(ks, src)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5): eng.keyswitch(ks, src)
    e1.record(); torch.cuda.synchronize()
    print('KS B=%d: %.3f ms' % (B, e0.elapsed_time(e1)/5))
