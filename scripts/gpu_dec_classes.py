"""Decoder latency per corpus class: one frame of ONE class per SM, then 32 per SM."""
import sys
from pathlib import Path
sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
import numpy as np, torch, ctypes as C
from zstd_jni_b200 import corpus, _native
from zstd_jni_b200.zstd import ZstdBatchContext
L = _native.lib()
ctx = ZstdBatchContext(0); ctx.setOption("timing", 1)
dev = torch.device("cuda:0")
sms = torch.cuda.get_device_properties(dev).multi_processor_count
stride = (L.ZSTD_compressBound(131072) + 32 + 63) // 64 * 64
buf = C.create_string_buffer(4096)
stream = torch.cuda.Stream(); st = stream.cuda_stream
counts = [int(a) for a in sys.argv[1:]] or [sms, 32 * sms]
for cls in range(8):
    for n in counts:
        data = np.stack([corpus.chunk(cls + 8 * (i % 64)) for i in range(n)])
        d_src = torch.from_numpy(data.reshape(-1)).to(dev)
        d_off = torch.arange(0, (n + 1) * 131072, 131072, dtype=torch.int64, device=dev)
        d_slots = torch.empty(n * stride, dtype=torch.uint8, device=dev); d_sizes = torch.zeros(n, dtype=torch.int64, device=dev)
        d_out = torch.empty(n * stride, dtype=torch.uint8, device=dev); d_ooff = torch.zeros(n + 1, dtype=torch.int64, device=dev)
        d_back = torch.zeros(n * 131072, dtype=torch.uint8, device=dev); d_res = torch.zeros(n, dtype=torch.int64, device=dev)
        L.zstdb200_compress_device(ctx.handle, 3, n, d_src.data_ptr(), d_off.data_ptr(), d_slots.data_ptr(), stride, d_sizes.data_ptr(), st)
        L.zstdb200_compact_device(ctx.handle, n, d_slots.data_ptr(), stride, d_sizes.data_ptr(), d_out.data_ptr(), d_ooff.data_ptr(), st)
        torch.cuda.synchronize()
        for rep in range(2):
            L.zstdb200_kernel_times(ctx.handle, buf, 4096)
            L.zstdb200_decompress_device(ctx.handle, n, d_out.data_ptr(), d_ooff.data_ptr(), d_back.data_ptr(), d_off.data_ptr(), d_res.data_ptr(), st)
            torch.cuda.synchronize()
        L.zstdb200_kernel_times(ctx.handle, buf, 4096)
        ok = bool(torch.equal(d_back, d_src))
        print(f"class {cls} n={n} ok={ok} csize/frame={int(d_ooff[-1])//n} | {buf.value.decode()}", flush=True)
