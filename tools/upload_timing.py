import sys, time
import os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, numpy as np
from of_dis_b200 import api, params, preprocess, synth
prm = params.operating_point(2, 1024)
i0, i1, _ = synth.synthetic_pair(436, 1024, 1, seed=0)
pyr = preprocess.PairPyramids(i0, i1, prm.sc_f, prm.p_samp_s)
B = 64
st = torch.cuda.Stream(); torch.cuda.set_stream(st)
ctx = api.Context(prm, pyr.width, pyr.height, pyr.imgpadding, B, stream=st.cuda_stream)
ff = ctx.packed_frame_floats; ni = ctx.packed_images_frame_floats
hin = torch.empty((B, ff), dtype=torch.float32).pin_memory()
for f in range(B): ctx.pack_frame(pyr, hin[f].numpy())
himg = torch.empty((B, ni), dtype=torch.float32).pin_memory(); himg.copy_(hin[:, :ni])
himg2 = torch.empty((B, ni), dtype=torch.float32, pin_memory=True); himg2.copy_(himg)
hbig = torch.empty((4 * B, ni), dtype=torch.float32, pin_memory=True); hbig.zero_()
def t(fn, n=30):
    for _ in range(5): fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(n): fn()
    b.record(st); torch.cuda.synchronize()
    return round(a.elapsed_time(b) / n, 4)
dfull = torch.empty((B, ff), dtype=torch.float32, device='cuda')
dimg2 = torch.empty((B, ni), dtype=torch.float32, device='cuda')
dbig = torch.empty((4 * B, ni), dtype=torch.float32, device='cuda')
small = torch.zeros(1024, device='cuda')
MBi = ni * 4 * B / 1e6; MBf = ff * 4 * B / 1e6
def rep(name, ms, mb): print('%-44s %.4f ms  %.1f GB/s' % (name, ms, mb / ms))
rep('torch himg->dimg2', t(lambda: dimg2.copy_(himg, non_blocking=True)), MBi)
rep('torch himg2->dimg2', t(lambda: dimg2.copy_(himg2, non_blocking=True)), MBi)
def alt():
    dimg2.copy_(himg, non_blocking=True); small.add_(1.0)
rep('torch himg->dimg2 + tiny kernel', t(alt), MBi)
rep('torch hin->dfull', t(lambda: dfull.copy_(hin, non_blocking=True)), MBf)
rep('torch hin[:B/2]->dfull[:B/2]', t(lambda: dfull[:B // 2].copy_(hin[:B // 2], non_blocking=True)), MBf / 2)
rep('torch hbig->dbig (4x)', t(lambda: dbig.copy_(hbig, non_blocking=True)), 4 * MBi)
rep('torch hbig[:B]->dbig[:B]', t(lambda: dbig[:B].copy_(hbig[:B], non_blocking=True)), MBi)
rep('ofdis upload_packed(hin)', t(lambda: ctx.upload_packed(0, B, hin.data_ptr())), MBf)
rep('ofdis upload_packed_images(himg)', t(lambda: ctx.upload_packed_images(0, B, himg.data_ptr())), MBi)
rep('ofdis upload_packed_images(himg2)', t(lambda: ctx.upload_packed_images(0, B, himg2.data_ptr())), MBi)
rep('ofdis upload_packed_images(hin as contiguous)', t(lambda: ctx.upload_packed_images(0, B, hin.data_ptr())), MBi)
rep('ofdis upload_packed_images(hbig)', t(lambda: ctx.upload_packed_images(0, B, hbig.data_ptr())), MBi)
rep('ofdis upload_packed_images(B/2, himg)', t(lambda: ctx.upload_packed_images(0, B // 2, himg.data_ptr())), MBi / 2)
rep('torch himg->dimg2 (again)', t(lambda: dimg2.copy_(himg, non_blocking=True)), MBi)
rep('torch hin->dfull (again)', t(lambda: dfull.copy_(hin, non_blocking=True)), MBf)
# D2H
hout = torch.empty((B, 436 * 1024 * 2 // 1), dtype=torch.float32, pin_memory=True)
dout = torch.empty_like(hout, device='cuda')
rep('torch D2H flow-sized', t(lambda: hout.copy_(dout, non_blocking=True)), hout.numel() * 4 / 1e6)
