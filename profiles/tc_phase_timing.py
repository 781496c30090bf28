import os, sys, ctypes as C
sys.path.insert(0, __import__("os").path.dirname(__import__("os").path.dirname(__import__("os").path.abspath(__file__))))
import torch, gnn_pathplanning_b200 as gp
from gnn_pathplanning_b200 import _lib
B,N,K=32768,10,3
w=((torch.rand(128,1,K,128)-0.5)*0.2).cuda(); b=(torch.rand(128,1)-0.5).cuda()
x=torch.randn(B,N,128,device="cuda"); S=torch.rand(B,N,N,device="cuda")*0.2
lib=_lib.load()
_lib.set_debug_option("gf_mode", 2); _lib.set_debug_option("tc_timing", 1)
for i in range(3): y=gp.graph_filter(x,S,w,b,True,gp.NODE_MAJOR,gp.NODE_MAJOR)
out=(C.c_ulonglong*6)()
lib.gpp_debug_tc_timing(out)
y=gp.graph_filter(x,S,w,b,True,gp.NODE_MAJOR,gp.NODE_MAJOR)
lib.gpp_debug_tc_timing(out)
v=list(out); tiles=v[5]
print("tiles(thread0 ctas)",tiles, "per-tile cycles: items %.0f mma-wait %.0f E1 %.0f E2 %.0f store+logits %.0f"%tuple(v[i]/tiles for i in range(5)))
