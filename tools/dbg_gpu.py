import sys, os, ctypes, numpy as np
ROOT=os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0,ROOT); sys.path.insert(0,ROOT+"/tests"); sys.path.insert(0,ROOT+"/tools")
import helpers, fuzzgen
from tokenizers_b200 import Tokenizer, _lib
from oracle import oracle as orc
from test_pretok_logic_cpu import _emul, _pack2
js=helpers.asset_json("gpt2_style")
tok=Tokenizer.from_str(js, device=0)
E=_emul()
tbl=_pack2(orc.class_table("onig"))
docs=fuzzgen.rand_docs(5000, 1500, max_len=300)
data,off=helpers.pack_docs(docs)
n=int(off[-1])
tok.pre_tokenize_batch(docs)
L=_lib.lib()
nch=min(n//32+1, 8192)
g=np.zeros(8192*8,dtype=np.uint32)
L.b2t_debug_k1.argtypes=[ctypes.c_void_p, ctypes.c_size_t]
print("rc", L.b2t_debug_k1(g.ctypes.data, g.size))
g=g.reshape(-1,8)
buf=np.concatenate([data,np.zeros(64,dtype=np.uint8)])
st=np.zeros(n//32+2,dtype=np.uint32); pl=np.zeros((n//32+2)*8,dtype=np.uint32)
E.b2t_emul_fast_planes.argtypes=[ctypes.c_void_p,ctypes.c_uint64,ctypes.c_void_p,ctypes.c_uint32,ctypes.c_void_p,ctypes.c_void_p,ctypes.c_void_p]
E.b2t_emul_fast_planes(buf.ctypes.data,n,off.ctypes.data,len(docs),tbl.ctypes.data,st.ctypes.data,pl.ctypes.data)
pl=pl.reshape(-1,8)
names=["lead","cont","L","N","S","SP","pL","start"]
shown=0
for c in range(nch):
    for k in range(8):
        a=int(g[c,k]); b=int(pl[c,k])
        if k==6: a>>=31; b>>=31
        if a!=b:
            print("chunk",c,"it",c//32,"lane",c%32,names[k],"gpu %08x emu %08x"%(a,b), bytes(data[max(0,c*32-8):c*32+40]))
            shown+=1
    if shown>16: break
print("done")
