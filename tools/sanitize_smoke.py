import sys; sys.path.insert(0,'.')
import numpy as np, opencorr_b200 as ob
from opencorr_b200 import synth
ref,tar=synth.speckle_pair_2d(200,180); xy=synth.grid_2d(30,30,6,5,22,25)
e=ob.Engine(0)
for r in (16,9):
    q=ob.make_poi2d(xy); e.set_images_2d(ref,tar); e.fftcc2d(q,r,r); e.icgn2d_prepare(); e.icgn2d1(q,r,r,0.001,10); q2=q.copy(); e.icgn2d2(q2,r,r,0.001,10)
    print('2d r',r, (q[:,16]>0).sum(), (q2[:,16]>0).sum())
off=np.ones((len(xy),2),np.float32); q=ob.make_poi2d(xy); e.fftcc2d(q,16,16); e.icgn2d_ex(1,q,16,16,0.001,10,off,False)
r3,t3=synth.speckle_pair_3d(64,60,56); xyz=synth.grid_3d(24,22,22,2,2,2,9,9,9)
for r in (16,7):
    if r==16: xyz2=np.array([[32,30,28]],np.float32)
    else: xyz2=xyz
    q=ob.make_poi3d(xyz2); e.set_images_3d(r3,t3); e.fftcc3d(q,r,r,r); e.icgn3d_prepare(); e.icgn3d1(q,r,r,r,0.001,20); print('3d r',r,q[:,18])
e.close(); print('done')
# round 2: a queue long enough to fill every SM with one-warp-per-POI ICGN2D1 CTAs and the chunked host-queue path,
# once with a pageable and once with a page-locked (zero-copy) queue; a group context of every visible device
import ctypes
from opencorr_b200 import _capi
lib=_capi.load()
ref,tar=synth.speckle_pair_2d(1024,1024); xy=synth.grid_2d(40,40,135,130,7,7)
e=ob.Engine(0); e.set_images_2d(ref,tar); e.icgn2d_prepare()
for pin in (0,1):
    q=ob.make_poi2d(xy)
    if pin: lib.ocb_host_register(ctypes.c_void_p(q.ctypes.data), q.nbytes)
    e.set_images_2d(ref,tar); e.fftcc2d(q,16,16); e.icgn2d_prepare(); e.icgn2d1(q,16,16,0.001,10)
    if pin: lib.ocb_host_unregister(ctypes.c_void_p(q.ctypes.data))
    print('long queue, pinned' if pin else 'long queue, pageable', len(q), (q[:,16]>0.9).sum())
e.close()
g=ob.Engine(list(range(lib.ocb_device_count()))); q=ob.make_poi2d(xy); g.set_images_2d(ref,tar); g.fftcc2d(q,16,16); g.icgn2d_prepare(); g.icgn2d1(q,16,16,0.001,10); print('group', g.member_count, (q[:,16]>0.9).sum()); g.close()
print('done round 2')
