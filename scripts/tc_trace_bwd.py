import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import __graft_entry__ as g; g.build()
from zeggs_b200 import ops, synth, _lib
from tests._util import make_decoder, stats_tensors, NAMES, tt
dev = torch.device("cuda:0"); st = stats_tensors()
H, B, T = int(os.environ.get("H", 1024)), int(os.environ.get("B", 32)), 40
P = synth.make_params(H=H, seed=3, with_style=False)
win = tt(synth.make_pose_windows(B, T, seed=3))
speech = (torch.randn(B, T, 64) * 0.5).to(dev).requires_grad_(True); style = torch.randn(B, 1, 64).repeat(1, T, 1)
dec = make_decoder(P, H, device=dev).train()
args = [win[n][:, 0].to(dev) for n in NAMES] + [win["gaze_pos"].to(dev), speech, style.to(dev), st["parents"]] + \
       [st[k].to(dev) for k in ("anim_input_mean", "anim_input_std", "anim_output_mean", "anim_output_std")] + [st["dt"]]
ops.set_decoder_engine("tc")
def run():
    out = dec(*args); sum(o.sum() for o in out).backward()
run(); torch.cuda.synchronize()
buf = torch.zeros(2 * 64 * 32, dtype=torch.int64, device=dev)     # [CTA 0, 1][reverse step][event], clock64 of each CTA's SM
out = dec(*args); loss = sum(o.sum() for o in out); torch.cuda.synchronize()
_lib.lib().zeggs_debug_set_tc_trace(buf.data_ptr())
loss.backward(); torch.cuda.synchronize()
_lib.lib().zeggs_debug_set_tc_trace(None)
tr = buf.cpu().numpy().reshape(2, 64, 32)
names = {0:"L:B4/R seen (G1 image ready)",3:"L:G1 issued",2:"L:B2 seen",5:"L:G0 issued",4:"L:B3 seen",7:"L:DPA issued",9:"M:B2 chain done",10:"M:B3 chain done",11:"M:B4 chain done",
         14:"E:d(B2) ready",16:"E:epi B2 done",17:"E:d(B3) ready",18:"E:epi B3 done",19:"E:d(B4) ready",20:"E:R done"}
# bytes each CTA streams per reverse step (decoder_bwd_tc.cu make_btgeom): its 64-row half of the 128-row images, a whole 32-row image
U = 4 if H // 4 <= 132 else 8
kbH, N2, FG = H // 64, 6 * U, (2 * U + 3 + 7) // 8 * 8
for rank in (0, 1):
    N3 = N2 + (1 + rank) * FG
    stages = {"B2": (0, 9, (64 + N2) * 128 * kbH), "B3": (2, 10, (64 + N3) * 128 * kbH), "B4": (4, 11, (32 + 16) * 128 * kbH)}
    print(f"CTA {rank} (rank {rank} of pair 0), H={H} U={U}")
    for s_ in (10,):
        t = tr[rank, s_]
        base = t[0]
        for ev in sorted(names, key=lambda e: t[e]):
            print(f"   {t[ev] - base:8d}  {names[ev]}")
        print(f"   step period: {tr[rank, s_ + 1, 0] - base} cycles")
        for st_name, (e0, e1, nbytes) in stages.items():
            cyc = t[e1] - t[e0]
            print(f"   {st_name}: barrier seen -> chain done {cyc:6d} cycles, {nbytes / 1024:.0f} KB, {nbytes / max(cyc, 1):.1f} B/clk")
