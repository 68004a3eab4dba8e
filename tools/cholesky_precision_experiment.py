import os, sys
import numpy as np, scipy.linalg as spla
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gp_oracle as O
f32=lambda a: np.asarray(a,dtype=np.float32)
def trunc_tf32(x):
    x=f32(x).copy(); v=x.view(np.uint32); v &= np.uint32(0xffffe000); return x
def split(x):
    h=trunc_tf32(x); l=trunc_tf32(f32(x)-h); return h.astype(np.float64), l.astype(np.float64)
def mm3(A,B):   # 3xTF32 product A @ B.T with exact accumulation (fp32 rounding of result)
    ah,al=split(A); bh,bl=split(B)
    return f32(al@bh.T + ah@bl.T + ah@bh.T).astype(np.float64)
def chol_blocked(K, mode, NB=128):
    A=f32(K).astype(np.float64).copy(); n=A.shape[0]
    for j0 in range(0,n,NB):
        j1=min(j0+NB,n)
        if j0>0:
            if mode=='tc': A[j0:,j0:j1]-= mm3(A[j0:,:j0], A[j0:j1,:j0])
            else: A[j0:,j0:j1]= f32(A[j0:,j0:j1]-f32(f32(A[j0:,:j0])@f32(A[j0:j1,:j0]).T))
        Ljj=np.linalg.cholesky(f32(A[j0:j1,j0:j1]).astype(np.float64)); Ljj=f32(Ljj).astype(np.float64)
        A[j0:j1,j0:j1]=Ljj
        if j1<n: A[j1:,j0:j1]=f32(spla.solve_triangular(Ljj, A[j1:,j0:j1].T, lower=True).T)
    return np.tril(A)
def run(D,N,M,noise,seed=0):
    rs=np.random.RandomState(seed)
    X=rs.rand(N,D); C=rs.rand(M,D); C[:10]=X[0]+1e-3*rs.randn(10,D)
    y=np.sin(3*X).sum(1); y=(y-y.mean())/y.std()
    h=(0.0,noise,1.0,rs.uniform(0.3,2.0,size=D))
    m,v,L,alpha=O.predict('Matern52',h,X,C,y)
    K=O.cov('Matern52',h[2],h[3],X)+noise*np.eye(N); Kx=O.cov('Matern52',h[2],h[3],X,C)
    ei=O._ei_from_moments(y.min(),m,np.sqrt(v))
    out={}
    for mode in ('fp32','tc'):
        Lm=chol_blocked(K,mode)
        beta=spla.solve_triangular(Lm,Kx,lower=True); a=spla.cho_solve((Lm,True),y-h[0])
        m2=Kx.T@a+h[0]; v2=h[2]*(1+1e-6)-np.sum(beta**2,0)
        ei2=O._ei_from_moments(y.min(),m2,np.sqrt(np.maximum(v2,1e-300)))
        out[mode]=(np.abs(Lm-L).max()/np.abs(L).max(), np.abs(v2-v).max(), np.abs(m2-m).max(), np.abs(ei2-ei).max()/ei.max(), abs(np.log(np.diag(Lm)).sum()-np.log(np.diag(L)).sum()))
    return out
for cfg in [(2,256,2000,1e-3),(4,1024,3000,1e-3),(8,512,3000,1e-3),(8,512,3000,1e-6),(20,1024,3000,1e-3)]:
    print(cfg)
    for k,vv in run(*cfg).items(): print('   %-5s dL %.1e  dvar %.1e  dmean %.1e  dEI/maxEI %.1e  dlogdet %.1e'%((k,)+vv))
