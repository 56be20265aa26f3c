import sys, time, numpy as np, scipy.sparse as sp, scipy.sparse.linalg as spla
import os
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from circuitscape_b200 import graph

def hash32(x):
    x = x.astype(np.uint64)
    x ^= x >> 16; x = (x * 0x7feb352d) & 0xffffffff; x ^= x >> 15; x = (x * 0x846ca68b) & 0xffffffff; x ^= x >> 16
    return x

def strength(A, theta):
    S = A.tocsr().copy(); S.setdiag(0); S.eliminate_zeros()
    S.data = np.abs(S.data)
    if theta > 0:
        rmax = np.maximum.reduceat(S.data, S.indptr[:-1][np.diff(S.indptr)>0]) if S.nnz else np.array([])
        mx = np.zeros(S.shape[0]); mx[np.diff(S.indptr)>0] = rmax
        rows = np.repeat(np.arange(S.shape[0]), np.diff(S.indptr))
        keep = S.data >= theta*mx[rows]
        S = sp.csr_matrix((S.data[keep], (rows[keep], S.indices[keep])), shape=S.shape)
        S = S.maximum(S.T).tocsr()   # symmetric
    return S

def nbmax(S, v):
    # max over neighbours incl self; v uint64
    rows = np.repeat(np.arange(S.shape[0]), np.diff(S.indptr))
    out = v.copy()
    np.maximum.at(out, rows, v[S.indices])
    return out

def mis2(S, dynamic=False, seed_hash=True):
    n = S.shape[0]
    deg = np.diff(S.indptr)
    ids = np.arange(n, dtype=np.uint64)
    h = hash32(np.arange(n)) & np.uint64(0x3ffffff)   # 26 bits
    state = np.where(deg>0, 1, 0).astype(np.uint64)
    rows = np.repeat(np.arange(n), deg)
    rounds = 0
    while (state==1).any():
        rounds += 1
        if dynamic:
            isout = (state==0).astype(np.int64)
            isout[deg==0] = 0
            c1 = np.zeros(n, dtype=np.int64); np.add.at(c1, rows, isout[S.indices])
            cnt = np.minimum(c1, 15).astype(np.uint64)
        else:
            cnt = np.zeros(n, dtype=np.uint64)
        key = (state << np.uint64(62)) | (cnt << np.uint64(58)) | (h << np.uint64(32)) | ids
        key[state==0] = ids[state==0]
        t1 = nbmax(S, key); t2 = nbmax(S, t1)
        und = state==1
        win = und & (t2==key)
        lose = und & ~win & ((t2>>np.uint64(62))==2)
        state[win] = 2; state[lose] = 0
    roots = state==2
    return roots, rounds

def assign(S, roots):
    n = S.shape[0]
    deg = np.diff(S.indptr)
    agg = -np.ones(n, dtype=np.int64); agg[roots] = np.arange(roots.sum())
    rows = np.repeat(np.arange(n), deg)
    for p in range(2):
        snap = agg.copy()
        cand = snap[S.indices] >= 0
        if p==0: cand &= roots[S.indices]
        need = (snap[rows] < 0) & cand
        r, c, w = rows[need], S.indices[need], S.data[need]
        # strongest: sort by (r, -w)
        o = np.lexsort((-w, r)); r, c = r[o], c[o]
        first = np.r_[True, r[1:]!=r[:-1]]
        agg[r[first]] = snap[c[first]]
    return agg

def greedy(S):
    n = S.shape[0]; ip, ix = S.indptr, S.indices
    agg = -np.ones(n, dtype=np.int64); nagg=0
    for i in range(n):
        if agg[i]>=0: continue
        nb = ix[ip[i]:ip[i+1]]
        if len(nb)==0: continue
        if (agg[nb]>=0).any(): continue
        agg[i]=nagg; agg[nb]=nagg; nagg+=1
    seeded=agg.copy()
    for i in range(n):
        if agg[i]>=0: continue
        nb = ix[ip[i]:ip[i+1]]; w=S.data[ip[i]:ip[i+1]]
        ok = seeded[nb]>=0
        if ok.any(): agg[i]=seeded[nb[ok][np.argmax(w[ok])]]
    for i in range(n):
        if agg[i]>=0: continue
        nb = ix[ip[i]:ip[i+1]]
        if len(nb)==0: continue
        agg[i]=nagg
        for c in nb:
            if agg[c]<0: agg[c]=nagg
        nagg+=1
    return agg

def rho_est(A, dinv):
    n=A.shape[0]; i=np.arange(n)
    x = np.where(dinv!=0, 1.0 + ((i*2654435761)%1024)/1024.0*np.where(i&1,1.0,-1.0), 0.0)
    rho_inf = (abs(A)@np.ones(n)*abs(dinv)).max()
    lam=0
    for _ in range(8):
        acc=A@x; lam=(x@acc)/((x*x/np.where(dinv!=0,dinv,1))[dinv!=0].sum()); y=dinv*acc; x=y/np.abs(y).max()
    return min(rho_inf, max(lam, 0.7*rho_inf))

def build(A, aggfun, max_coarse=200, max_levels=12):
    levels=[]
    while True:
        d=A.diagonal(); dinv=np.where(d!=0,1/np.where(d!=0,d,1),0)
        rho=rho_est(A,dinv); om=(4/3)/rho
        L=dict(A=A,omega=om)
        levels.append(L)
        n=A.shape[0]
        if n<=max_coarse or len(levels)>=max_levels: break
        agg=aggfun(A, len(levels)-1)
        nagg=agg.max()+1
        if nagg<=0 or nagg>=n: break
        keep=agg>=0
        cnt=np.bincount(agg[keep],minlength=nagg).astype(float)
        T=sp.csr_matrix((1/np.sqrt(cnt[agg[keep]]),(np.nonzero(keep)[0],agg[keep])),shape=(n,nagg))
        P=(T-om*(sp.diags(dinv)@(A@T))).tocsr()
        R=P.T.tocsr(); Ac=(R@A@P).tocsr()
        if Ac.nnz>A.nnz: break
        L['P']=P; L['R']=R; L['nagg']=nagg
        A=Ac
    Ac=levels[-1]['A'].toarray()
    pinv=np.linalg.pinv(Ac, hermitian=True) if Ac.shape[0]<=320 else None
    return levels,pinv

import test_amg_host as T

def evaluate(name, A, aggfun, npairs=3):
    n=A.shape[0]; nodes=graph.focal_nodes(n,4,seed=7)
    t=time.time(); levels,pinv=build(A,aggfun); tb=time.time()-t
    opc=sum(l['A'].nnz for l in levels)/A.nnz
    its=[]
    for a in range(npairs):
        b=np.zeros(n); b[nodes[a]]=-1; b[nodes[a+1]]=1
        x,it=T.pcg(A,b,lambda r:T.vcycle(levels,pinv,r)); its.append(it)
    print(f"{name:34s} levels {[l['A'].shape[0] for l in levels]} opc {opc:.3f} iters {its} ({tb:.1f}s)", flush=True)

def mats(N):
    A,_=graph.synthetic_raster_laplacian(N,N,seed=42); yield 'uniform',A.tocsr()
    rng=np.random.default_rng(2); g=1.0/np.exp(rng.normal(0,1.5,(N,N))); g[rng.random(g.shape)<0.05]=0
    nm=graph.construct_node_map(g); G=graph.laplacian(graph.construct_graph(g,nm,False,False))
    big=max(graph.connected_components(G),key=len)-1; yield 'lognormal',G[big][:,big].tocsr()

if __name__=='__main__':
    N=int(sys.argv[1]) if len(sys.argv)>1 else 300
    for kind,A in mats(N):
        print('==',kind,N)
        evaluate('greedy', A, lambda A,l: greedy(strength(A,0)))
        for dyn in (False, True):
            for th in (0.0, 0.25, 0.5):
                def f(A,l,dyn=dyn,th=th):
                    S=strength(A,th); r,rounds=mis2(S,dynamic=dyn); 
                    if l==0: f.rounds=rounds; f.dens=r.sum()/A.shape[0]
                    return assign(S,r)
                evaluate(f'mis2 dyn={dyn} theta={th}', A, f)
                print('    L0 rounds',f.rounds,'1/density %.1f'%(1/f.dens))
