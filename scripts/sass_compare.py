#!/usr/bin/env python
"""Compares the SASS instruction stream of every kernel in two builds of libxtuner_b200.so (function by function,
addresses stripped).  Used to show that adding or removing template variants left the GPU-validated default kernels
untouched:   python scripts/sass_compare.py OLD.so NEW.so"""
import subprocess, re, hashlib, sys
def funcs(lib):
    out = subprocess.run(["cuobjdump","-sass",lib],capture_output=True,text=True).stdout
    res={}; cur=None
    for line in out.splitlines():
        m=re.search(r"Function : (\S+)", line)
        if m: cur=m.group(1); res[cur]=[]; continue
        m=re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(.*?);", line)
        if m and cur: res[cur].append(m.group(1).strip())
    return res
old=funcs(sys.argv[1]); new=funcs(sys.argv[2])
def demangle(n): return subprocess.run(["c++filt",n],capture_output=True,text=True).stdout.strip().split("(")[0]
newd={demangle(k):k for k in new}
def dropped(d):  # a template parameter removed together with its other value: <M, N, E, 1> -> <M, N, E>, f<true> -> f
    d=re.sub(r"<(\d+), (\d+), (\d+), 1>$", r"<\1, \2, \3>", d)
    d=re.sub(r"(::rmsnorm_gate_kernel<\d+, \d+, \d+), true>$", r"\1>", d)  # the gate became unconditional
    d=re.sub(r"(::dispatch_bwd_rmsnorm_kernel)<0, (\d+)>$", r"\1<\2>", d)  # runtime K only: KT = 0 went
    return re.sub(r"^void (\S+)<true>$", r"\1", d)
same=diff=0
for k,v in old.items():
    d=demangle(k)
    cands=[nk for nd,nk in newd.items() if nd in (d, dropped(d)) or nd.replace(", false>",">")==d or nd.replace(", (bool)0>",">")==d
           or re.sub(r"^void (\S+)<false>$", r"\1", nd)==d]  # a kernel that became a template over an off-by-default switch
    if not cands:
        print("MISSING in new:", d); continue
    nv=new[cands[0]]
    if v==nv: same+=1
    else:
        diff+=1
        # opcode histogram diff
        import collections
        ho=collections.Counter(x.split()[0].split('.')[0] if not x.startswith('@') else x.split()[1].split('.')[0] for x in v)
        hn=collections.Counter(x.split()[0].split('.')[0] if not x.startswith('@') else x.split()[1].split('.')[0] for x in nv)
        delta={op:hn[op]-ho[op] for op in set(ho)|set(hn) if hn[op]!=ho[op]}
        print(f"DIFF {d}: {len(v)} -> {len(nv)} instrs; opcode delta {delta}")
print("identical:",same,"different:",diff)
