import sys, time
import os; sys.path[:0] = [os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests')]
import numpy as np, recipes
from oracle import brnn_oracle
D,K,H,N,tl,T,L,B = 41,32,1024,3,2,800,100,2
datas, labelss = recipes.synth_batch(D, K, [T]*B, [L]*B, seed=33)
rel=lambda a,b: np.linalg.norm(a-b)/np.linalg.norm(b)
def run(noise):
    np.random.seed(33)
    on = brnn_oracle.NNet(D,K,H,N,T,temporalLayer=tl,dtype=np.float64); on.initParams()
    if noise:
        rng = np.random.RandomState(1)
        class NoisyW(np.ndarray):
            pass
        # emulate a forward GEMM whose outputs carry a relative error `noise`: perturb the layer inputs->outputs by wrapping forward
        orig = on.forward
        def fwd(data):
            hActs, For, Back, probs = orig(data)
            return hActs, For, Back, probs
        # simplest faithful emulation: perturb the weights' products by perturbing activations is intrusive; instead perturb the
        # biases per frame is not possible -> perturb the INPUT features relatively (propagates like a first-layer GEMM error)
        return on, rng
    return on, None
on,_ = run(0)
c0,g0,_ = on.costAndGradBatch(datas, labelss)
g0=[(dw.copy(),db.copy()) for dw,db in g0]
for noise in (1e-7, 1e-6, 1e-5):
    rng=np.random.RandomState(1)
    nd=[d*(1+noise*rng.randn(*d.shape)).astype(np.float32) for d in datas]
    nd=[x.astype(np.float32) for x in nd]
    np.random.seed(33)
    on2 = brnn_oracle.NNet(D,K,H,N,T,temporalLayer=tl,dtype=np.float64); on2.initParams()
    c,g,_ = on2.costAndGradBatch(nd, labelss)
    print('input noise %.0e: cost rel %.1e'%(noise, np.max(np.abs(c-c0)/c0)), ['%.1e'%rel(dw,odw) for (dw,db),(odw,odb) in zip(g,g0)])
