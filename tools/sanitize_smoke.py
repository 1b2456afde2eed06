"""Small forward of every entry point, for compute-sanitizer (memcheck) on the GPU box. Test infrastructure."""
import os, sys
import numpy as np
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wav2lip_b200 import audio
from wav2lip_b200.models import SyncNet_color, Wav2Lip, Wav2Lip_disc_qual

torch.manual_seed(0)
with torch.no_grad():
    g = Wav2Lip().cuda().eval()
    y = g(torch.rand(3, 1, 80, 16).cuda(), torch.rand(3, 6, 96, 96).cuda())
    y5 = g(torch.rand(2, 2, 1, 80, 16).cuda(), torch.rand(2, 6, 2, 96, 96).cuda())
    y6 = g(torch.rand(6, 1, 80, 16).cuda(), torch.rand(6, 6, 96, 96).cuda())   # enough tiles for the patch kernels
    ys = list(g.infer_stream(iter([(torch.rand(5, 1, 80, 16), torch.rand(5, 6, 96, 96)),
                                   (torch.rand(2, 1, 80, 16), torch.randint(0, 256, (2, 96, 96, 3), dtype=torch.uint8))])))
    u = g.infer_u8(torch.rand(3, 1, 80, 16).cuda(), torch.randint(0, 256, (3, 96, 96, 3), dtype=torch.uint8).cuda())
    s = SyncNet_color().cuda().eval()
    a, v = s(torch.rand(3, 1, 80, 16).cuda(), torch.rand(3, 15, 48, 96).cuda())
    d = Wav2Lip_disc_qual().cuda().eval()
    p = d(torch.rand(2, 3, 2, 96, 96).cuda())
    m = audio.melspectrogram(np.random.randn(5000).astype(np.float32))
    c = audio.mel_chunks(m, 25.0)
    ms = audio.melspectrogram(np.random.randn(57).astype(np.float32))           # multi-fold reflect padding
    # scope row f2: crop + resize, paste, the whole inner loop in one call
    frames = torch.randint(0, 256, (2, 72, 88, 3), dtype=torch.uint8).cuda()
    boxes = [[0, 5, 60, 7, 80], [1, 0, 72, 0, 88]]
    cr = g.crop_resize(frames, boxes)
    pa = g.paste(u[:2], frames, boxes)
    fr = g.infer_frames(torch.rand(2, 1, 80, 16).cuda(), frames, boxes)
    # streaming: the ring mel kernel (host and device pieces, a wrapping 2^11 ring, the end reflection), the chunk
    # gather, and a session step uncaptured and replayed from its graph
    msr = audio.MelStream(0, 11)
    mw = np.random.randn(7000).astype(np.float32)
    mparts = [msr.push(mw[:3000]), msr.push(torch.from_numpy(mw[3000:6100]).cuda()).cpu().numpy(), msr.finish()]
    from wav2lip_b200.stream import LipSyncSession
    sess = LipSyncSession(g, frames, 25.0, rects=[(7, 5, 80, 60), (0, 0, 88, 62)], batch=2)
    sfr = [sess.push(np.random.randn(3200).astype(np.float32))[1] for _ in range(3)] + [sess.finish()[1]]
    sess.close()
    # a stream group: the audio scatter (host and device pieces), the multi-ring mel kernel, and steps of two bucket
    # sizes (a padding row, frames of two sizes, one not 16-byte aligned) uncaptured and replayed
    from wav2lip_b200.stream import LipSyncServer
    srv = LipSyncServer(g, max_batch=4, audio_ring_log2=11)
    frames2 = torch.randint(0, 256, (3, 57, 91, 3), dtype=torch.uint8).cuda()
    ga = srv.open(frames, 25.0, rects=[(7, 5, 80, 60), (0, 0, 88, 62)])
    gb = srv.open(frames2, 29.97, box=(3, 50, 5, 80))
    gw = np.random.randn(9000).astype(np.float32)
    gfr = [srv.tick({ga: gw[k:k + 1500], gb: torch.from_numpy(gw[k:k + 1500]).cuda()}) for k in range(0, 6000, 1500)]
    gfr.append(srv.tick({ga: gw[6000:]}, finish=[ga, gb]))
    srv.close()
    # many units of 128-channel tiles: a 128-channel residual block and a transposed-conv phase set
    from wav2lip_b200.models.conv import Conv2d, Conv2dTranspose
    sw = Conv2d(128, 128, 3, 1, 1, residual=True).cuda().eval()(torch.rand(140, 128, 24, 24).cuda())
    swt = Conv2dTranspose(320, 128, 3, 2, 1, 1).cuda().eval()(torch.rand(150, 320, 12, 12).cuda())
    # scope row f4: the S3FD detector network
    from wav2lip_b200.face_detection.detection.sfd.net_s3fd import s3fd
    det = s3fd().cuda().eval()
    dm = det(torch.rand(1, 3, 96, 128).cuda() * 255)
    torch.cuda.synchronize()
# scope row f1: one training iteration through the autograd bridge and one fused native step (B=1, T=5)
from wav2lip_b200.training import Wav2LipTrainStep
gt_ = Wav2Lip().cuda().train()
out = gt_(torch.rand(2, 1, 80, 16).cuda(), torch.rand(2, 6, 96, 96).cuda())
out.mean().backward()
ex = SyncNet_color().cuda().train()
step = Wav2LipTrainStep(Wav2Lip().cuda().train(), ex, lr=1e-4, syncnet_wt=0.03)
ls = step(torch.rand(1, 6, 5, 96, 96).cuda(), torch.rand(1, 5, 1, 80, 16).cuda(), torch.rand(1, 1, 80, 16).cuda(), torch.rand(1, 3, 5, 96, 96).cuda())
torch.cuda.synchronize()
print("train ok", [float(v) for v in ls.cpu()])
print("ok", y.shape, y5.shape, u.shape, a.shape, p.shape, m.shape, c.shape, float(y.mean()), float(p.mean()))
