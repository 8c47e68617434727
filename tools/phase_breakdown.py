import sys, torch
import os; sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from genefaceplusplus_b200 import _capi, scene as scn
from genefaceplusplus_b200.renderer import RADNeRFTorso
prec = sys.argv[1] if len(sys.argv)>1 else 'fp16'
if '--one-cta' in sys.argv: os.environ['GFPP_ONE_CTA'] = '1'   # phase timings without the co-resident CTA
sc = scn.Scene(H=512,W=512,T=20,torso=True,density_scale=8.0)
m = RADNeRFTorso(sc.hparams); m.load_state_dict(sc.state); m.density_scale=8.0; m.mlp_precision=prec; m=m.cuda().eval()
poses = torch.stack([sc.pose(t) for t in range(20)])
kw=dict(cond_seq=sc.cond,bg_color=sc.bg_color,bg_coords=sc.bg_coords,T_thresh=0.01,frames_per_call=20)
m.render_clip(poses, sc.intrinsics,512,512,**kw); torch.cuda.synchronize()
buf = torch.zeros(32,dtype=torch.int64,device='cuda')
_capi.lib().gfpp_profile_phases(buf.data_ptr())
m.render_clip(poses, sc.intrinsics,512,512,**kw); torch.cuda.synchronize()
_capi.lib().gfpp_profile_phases(None)
v = buf.cpu().tolist(); nb = v[31]
if not os.environ.get('GFPP_HEAD_V1') and prec in ('fp16', 'robust'):   # row-owner kernel: stamps of row 0 of slot 0 of every CTA
    # PH(i) index -> phase of csrc/head_v2_kernel.cu (16-18 are not stamped; sigma L2's geo rows are folded into col L0).
    # Ambient out and colour out run in the epilogues that feed them: 4 and 14 time their mma.sync and the owners' barrier; the
    # sigma row runs under colour L0's MMAs, inside 13. fp16 stamps 6 (its owners wait for the gather warp) and only the position
    # levels below GATHER_L0 as 8 / 10; robust stamps 8 and 10, not 6
    names2 = {6: 'wait for staged position features', 0: 'operand rows (pos feats, cond, SH)', 12: 'fate + march', 1: 'refill',
              2: 'MMA + epi amb L0', 3: 'MMA amb L1', 4: 'amb out (mma.sync) + hand-over', 5: 'tanh', 7: 'ambient gather',
              8: 'prefetch pos levels 0-7', 9: 'MMA + epi sig L0', 10: 'prefetch pos levels 8-15', 11: 'MMA + epi sig L1',
              13: 'MMA col L0 (+ sigma row under it)', 14: 'col out (mma.sync) + hand-over', 15: 'sigmoid',
              19: 'composite + batch check'}
    tot = sum(v[i] for i in names2)
    print(f'precision {prec} (v2): batches of slot 0 {nb}, cycles per batch of one slot = {tot/nb:.0f}')
    for i, n in names2.items(): print(f'  {n:32s} {v[i]/nb:9.0f} cyc/batch  {100*v[i]/tot:5.1f}%')
    sys.exit(0)
tot=sum(v[:11])
names=['refill+publish','pos gather+cond','MMA amb0','epi amb0','MMA amb1','epi amb1','narrow amb + tanh','amb gather','sigma net (3 MMA+3 epi)','color net (2 MMA + epi)','composite+march']
print(f'precision {prec}: batches {nb}, cycles/batch (thread 0 of each CTA) = {tot/nb:.0f}')
for n,c in zip(names,v[:11]): print(f'  {n:28s} {c/nb:9.0f} cyc/batch  {100*c/tot:5.1f}%')
