#!/usr/bin/env python
"""Standalone GPU sanity checks needs an H100 before the test-suite: each check runs in its
own subprocess under a timeout so a hung kernel cannot take the whole gpurun call down.

    python tools/gpu_check.py [gemm|bn|all]   -> writes gpurun_out/gpu_check.json
"""
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CHECKS = {
    "gemm_tn": """
import torch; from edl_b200 import ops
torch.manual_seed(0)
for (m,n,k) in [(128,128,64),(128,128,256),(300,128,64),(1568,2048,512),(257,64,256),(32,1000,2048)]:
    a=torch.randn(m,k,device='cuda').bfloat16(); b=torch.randn(n,k,device='cuda').bfloat16()
    d=ops.gemm_bf16(a,b); torch.cuda.synchronize()
    ref=a.float()@b.float().t()
    print('tn',m,n,k,'rel',((d.float()-ref).norm()/ref.norm()).item())
""",
    "gemm_bmn": """
import torch; from edl_b200 import ops
torch.manual_seed(0)
for (m,n,k) in [(128,128,64),(300,128,64),(1568,512,2048),(500,64,256)]:
    a=torch.randn(m,k,device='cuda').bfloat16(); b=torch.randn(k,n,device='cuda').bfloat16()
    d=ops.gemm_bf16(a,b,b_mn_major=True); torch.cuda.synchronize()
    ref=a.float()@b.float()
    print('bmn',m,n,k,'rel',((d.float()-ref).norm()/ref.norm()).item())
""",
    "gemm_wgrad": """
import torch; from edl_b200.ops import gemm as G
torch.manual_seed(0)
for (m,n,k,s) in [(128,128,64,1),(256,64,1000,4),(512,128,6272,16),(1000,2048,32,1)]:
    a=torch.randn(k,m,device='cuda').bfloat16(); b=torch.randn(k,n,device='cuda').bfloat16()
    out=G._wgrad_impl(a,b,(m,n),None,split_k=s); torch.cuda.synchronize()
    ref=a.float().t()@b.float()
    print('wgrad',m,n,k,s,'rel',((out.float()-ref).norm()/ref.norm()).item())
""",
    "gemm_stats": """
import torch; from edl_b200 import ops
torch.manual_seed(0)
m,n,k=777,256,128
a=torch.randn(m,k,device='cuda').bfloat16(); b=torch.randn(n,k,device='cuda').bfloat16()
st=torch.zeros(2*n,device='cuda'); sc=torch.rand(n,device='cuda')+0.5; sh=torch.randn(n,device='cuda')
d=ops.gemm_bf16(a,b,col_scale=sc,col_shift=sh,relu=True,col_stats=st); torch.cuda.synchronize()
ref=torch.relu((a.float()@b.float().t())*sc+sh)
print('epi rel',((d.float()-ref).norm()/ref.norm()).item(), 'stats', ((st[:n]-d.float().sum(0)).norm()/d.float().sum(0).norm()).item())
""",
    "bn": """
import torch; from edl_b200 import ops
x=torch.randn(8,64,28,28,device='cuda').bfloat16().contiguous(memory_format=torch.channels_last).requires_grad_(True)
g=torch.ones(64,device='cuda',requires_grad=True); b=torch.zeros(64,device='cuda',requires_grad=True)
y=ops.batch_norm_act(x,g,b,torch.zeros(64,device='cuda'),torch.ones(64,device='cuda'),relu=True)
y.float().sum().backward(); torch.cuda.synchronize()
print('bn mean',y.float().mean().item(),'dx',x.grad.float().abs().mean().item())
""",
}


def main():
    which = sys.argv[1] if len(sys.argv) > 1 else "all"
    out_dir = os.path.join(ROOT, "gpurun_out")
    os.makedirs(out_dir, exist_ok=True)
    results = {}
    for name, code in CHECKS.items():
        if which != "all" and not name.startswith(which):
            continue
        t0 = time.time()
        try:
            r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n%s" % (ROOT, code)],
                               capture_output=True, text=True, timeout=120)
            results[name] = {"rc": r.returncode, "out": r.stdout[-3000:], "err": r.stderr[-3000:],
                             "secs": time.time() - t0}
        except subprocess.TimeoutExpired as e:
            results[name] = {"rc": "TIMEOUT", "out": (e.stdout or b"")[-2000:].decode("utf8", "replace")
                             if isinstance(e.stdout, bytes) else str(e.stdout)[-2000:], "secs": time.time() - t0}
        print("==", name, results[name]["rc"])
        print(results[name].get("out", ""))
        if results[name]["rc"] != 0:
            print(results[name].get("err", "")[-1500:])
    with open(os.path.join(out_dir, "gpu_check.json"), "w") as fh:
        json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
