"""k_parse latency of a lone warp per corpus class: one frame of ONE class per SM, then 32 per SM (a full wave)."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np, torch, ctypes as C
from zstd_jni_b200 import corpus, _native
from zstd_jni_b200.zstd import ZstdBatchContext
L = _native.lib()
level = int(sys.argv[1]) if len(sys.argv) > 1 else 3
ctx = ZstdBatchContext(0); ctx.setOption("timing", 1)
dev = torch.device("cuda:0")
sms = torch.cuda.get_device_properties(dev).multi_processor_count
stride = (L.ZSTD_compressBound(131072) + 32 + 63) // 64 * 64
buf = C.create_string_buffer(4096)
stream = torch.cuda.Stream(); st = stream.cuda_stream
for cls in range(8):
    for n in (sms, 32 * sms):
        data = np.stack([corpus.chunk(cls + 8 * (i % 64)) for i in range(n)])
        d_src = torch.from_numpy(data.reshape(-1)).to(dev)
        d_off = torch.arange(0, (n + 1) * 131072, 131072, dtype=torch.int64, device=dev)
        d_slots = torch.empty(n * stride, dtype=torch.uint8, device=dev)
        d_sizes = torch.zeros(n, dtype=torch.int64, device=dev)
        for rep in range(2):
            L.zstdb200_compress_device(ctx.handle, level, n, d_src.data_ptr(), d_off.data_ptr(), d_slots.data_ptr(), stride, d_sizes.data_ptr(), st)
            torch.cuda.synchronize()
        L.zstdb200_kernel_times(ctx.handle, buf, 4096)
        print(f"class {cls} n={n} csize/frame={int(d_sizes.sum())//n} | {buf.value.decode()}", flush=True)
