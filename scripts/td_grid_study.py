"""CPU-only study (numpy restatement of the batched t-digest update of DESIGN.md §2; not used by the product or the tests): how
far is the digest's p50 / p95 / p99 from the EXACT sample quantile on log-normal streams (sigma 1.2 / 1.5, n = 10 K .. 1 M, 1 or 8
batches), for the shipped K_1 unit grid and for tail-weighted grids with the same number of cells?

    python scripts/td_grid_study.py
"""
import numpy as np, sys
THR=np.array([1,10,30,60,100,150,200,300,450,700,1000,3000,15000])
def td_code(v):
    v=v.astype(np.uint64); out=v.copy()
    big=v>=32
    lg=np.floor(np.log2(np.maximum(v,1).astype(np.float64))).astype(np.int64)
    # fix rounding
    lg=np.where((1<<lg.astype(np.uint64))>v, lg-1, lg); lg=np.where((1<<(lg+1).astype(np.uint64))<=v, lg+1, lg)
    sh=(lg-5).clip(0)
    code=((sh+1)<<5)|((v>>sh.astype(np.uint64))&31).astype(np.int64)
    return np.where(big,code,v.astype(np.int64))
def bucket(ms):
    b=1+np.searchsorted(THR,ms,side='left')  # count of thr < ms  => ms>thr
    return np.where(ms>=15001,14,b)
def items_of(vals):
    b=td_code(vals)+bucket(vals//1000)
    cnt=np.bincount(b,minlength=848); s=np.bincount(b,weights=vals.astype(np.float64),minlength=848)
    nz=cnt>0
    return s[nz]/cnt[nz], cnt[nz].astype(np.int64)
def compress(m,w,qtab):
    W=w.sum(); pref=np.cumsum(w)-w
    T=(qtab*float(W)).astype(np.uint64).astype(np.int64); T[-1]=W
    d=len(qtab)-1
    cell=np.searchsorted(T[1:d],pref,side='right')  # number of T_{c+1} <= pref
    # unique cells
    cw=np.bincount(cell,weights=w,minlength=d); cs=np.bincount(cell,weights=m*w,minlength=d)
    nz=cw>0
    return cs[nz]/cw[nz], cw[nz].astype(np.int64)
def add_batch(td,vals,qtab):
    m,w=items_of(vals)
    if td is None: mm,ww=m,w; mn,mx=vals.min(),vals.max()
    else:
        om,ow,mn,mx=td
        mm=np.concatenate([om,m]); ww=np.concatenate([ow,w]); o=np.argsort(mm,kind='stable'); mm=mm[o]; ww=ww[o]
        mn=min(mn,vals.min()); mx=max(mx,vals.max())
    cm,cw=compress(mm,ww,qtab)
    return cm,cw,mn,mx
def quantile(td,q):
    m,w,mn,mx=td; tot=w.sum(); target=q*tot
    cum=np.cumsum(w)-w; cen=cum+w/2.0
    i=np.searchsorted(cen,target,side='right')
    if i==0: pc,pm=0.0,float(mn); c,mean=cen[0],m[0]
    elif i==len(m): pc,pm=cen[-1],m[-1]; c,mean=float(tot),float(mx)
    else: pc,pm=cen[i-1],m[i-1]; c,mean=cen[i],m[i]
    span=c-pc
    return pm+(mean-pm)*((target-pc)/span) if span>0 else mean
def exact(v,q):
    v=np.sort(v); return float(v[min(len(v)-1,max(0,int(np.ceil(q*len(v)))-1))])
def k1(d):
    j=np.arange(d+1); q=0.5*(np.sin(np.pi*(j/d-0.5))+1); q[0]=0;q[-1]=1; return q
def piecewise(d, knots, fracs):
    # knots: q breakpoints [0,...,1]; fracs: fraction of cells per segment
    cells=np.round(np.array(fracs)*d).astype(int); cells[-1]+=d-cells.sum()
    q=[0.0]
    for a,b,c in zip(knots[:-1],knots[1:],cells):
        q+=list(a+(b-a)*np.arange(1,c+1)/c)
    q=np.array(q); q[-1]=1.0; return q
def evaluate(qtab,label,seeds=6):
    res={}
    for sigma in (1.2,1.5):
        for n in (10_000,20_000,50_000,100_000,300_000,1_000_000):
            for nb in (1,8):
                errs=[]
                for seed in range(seeds):
                    rng=np.random.default_rng(seed*1000+n%977+int(sigma*10))
                    v=np.minimum(rng.lognormal(np.log(20000),sigma,n),9e8).astype(np.uint32)+1
                    td=None
                    for part in np.array_split(v,nb): td=add_batch(td,part,qtab)
                    e=[abs(quantile(td,q)-exact(v,q))/exact(v,q) for q in (0.5,0.95,0.99)]
                    errs.append(e)
                errs=np.array(errs)
                res[(sigma,n,nb)]=errs.max(0)
    print(label)
    for k,v in res.items(): print(' ',k,' '.join(f'{x*100:.2f}' for x in v), ' ncent=',)
    worst=np.array(list(res.values())).max(0)
    print('  WORST p50/p95/p99 %:',' '.join(f'{x*100:.2f}' for x in worst))
    return res
def smooth(d, wa, w1, e1):
    """cells per unit q = wa + c1 / (1 - q + e1)^2 (wa uniform cells + w1 cells towards the upper tail), boundaries by bisection"""
    c1 = w1 / (1 / e1 - 1 / (1 + e1))
    K = lambda q: wa * q + c1 * (1 / (1 - q + e1) - 1 / (1 + e1))
    qs = [0.0]
    for j in range(1, d):
        lo, hi = 0.0, 1.0
        for _ in range(64):
            mid = 0.5 * (lo + hi)
            if K(mid) < j: lo = mid
            else: hi = mid
        qs.append(hi)
    return np.array(qs + [1.0])


if __name__=='__main__':
    evaluate(k1(200),'K_1, delta = 200 (shipped)', seeds=8)
    evaluate(piecewise(200,[0,.3,.7,.9,.975,1],[.05,.15,.15,.25,.40]),'piecewise: 40 % of the cells in q > 0.975', seeds=8)
    evaluate(smooth(200,80,120,.02),'smooth: 80 uniform cells + 120 cells ~ 1/(1.02 - q)^2', seeds=8)
