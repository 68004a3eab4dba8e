import os, sys
import numpy as np, scipy.linalg as spla
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import gp_oracle as O
def rnd_bits(x, bits):  # round to `bits` mantissa bits (incl. implicit) -- emulate tf32(11)/bf16(8)
    m, e = np.frexp(x); s = 2.0**bits
    return np.ldexp(np.round(m*s)/s, e)
def split(x, bits, pieces):
    out=[]; r=x.copy()
    for _ in range(pieces):
        p=rnd_bits(r,bits); out.append(p); r=r-p
    return out
def run(D,N,M,noise,kind='Matern52',seed=0, lsr=(0.3,2.0)):
    rs=np.random.RandomState(seed)
    X=rs.rand(N,D); C=rs.rand(M,D); C[:10]=X[0]+1e-3*rs.randn(10,D)
    y=np.sin(3*X).sum(1); y=(y-y.mean())/y.std()
    h=(0.0,noise,1.0,rs.uniform(*lsr,size=D))
    m,v,L,alpha=O.predict(kind,h,X,C,y)
    Kx=O.cov(kind,h[2],h[3],X,C)
    Linv=spla.solve_triangular(L,np.eye(N),lower=True)
    best=y.min()
    ei=O._ei_from_moments(best,m,np.sqrt(v))
    res={}
    f32=lambda a:a.astype(np.float32).astype(np.float64)
    # baseline: fp32 everything (inputs rounded to fp32, exact products)
    for name,(bits,pa,pb,terms) in {'fp32in':(24,1,1,[(0,0)]),'tf32x1':(11,1,1,[(0,0)]),'3xtf32':(11,2,2,[(0,0),(0,1),(1,0)]),
        'bf16x2_3':(8,2,2,[(0,0),(0,1),(1,0)]),'bf16x3_6':(8,3,3,[(0,0),(0,1),(1,0),(0,2),(1,1),(2,0)]),'bf16x3_3':(8,3,3,[(0,0),(0,1),(1,0)])}.items():
        A=split(f32(Linv),bits,pa); B=split(f32(Kx),bits,pb)
        beta=sum(A[i]@B[j] for i,j in terms)
        v2=h[2]*(1+1e-6)-np.sum(f32(beta)**2,axis=0)
        ei2=O._ei_from_moments(best,m,np.sqrt(np.maximum(v2,1e-300)))
        res[name]=(np.abs(v2-v).max(), np.abs(ei2-ei).max()/ei.max(), int(np.argmax(ei2)==np.argmax(ei)), (v2<=0).sum())
    return v.min(), res
for cfg in [(2,200,2000,1e-3),(8,512,3000,1e-3),(8,512,3000,1e-6),(20,1024,3000,1e-3),(4,1024,3000,1e-3),(32,1500,2000,1e-3)]:
    vmin,res=run(*cfg)
    print(cfg,'vmin %.2e'%vmin)
    for k,(dv,dei,am,neg) in res.items(): print('   %-9s max|dv| %.2e  max|dEI|/maxEI %.2e argmax_ok %d neg %d'%(k,dv,dei,am,neg))
