"""Diagnostic: determinism of the front end (G_pre) and its equality with the front end inside G_pipe."""
import os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from celebbasis_b200 import ops, synth, workload
from celebbasis_b200.tokenizer import SyntheticCLIPTokenizer
from celebbasis_b200.train_step import CelebBasisStep
from celebbasis_b200.step_graph import StepGraphs
from oracle import torch_ref
dev = torch.device("cuda:0")
kind = sys.argv[1] if len(sys.argv) > 1 else "tiny"
params = workload.model_params(kind)
om = torch_ref.OracleModel(params, clip_layers=workload.clip_layers(kind))
sd = synth.synth_state_dict(om, seed=0)
eng = CelebBasisStep(params, sd, synth.synth_celeb_basis(seed=0), dev, tokenizer=SyntheticCLIPTokenizer())
hw = workload.image_hw(kind)
G = StepGraphs(eng, B=1, T=77, n_chunks=2, image_hw=hw)
bs = [workload.synth_batch(kind, B=1, seed=1234, step=i) for i in range(2)]
b0, d0 = bs[0]
ids, mp, _ = eng.prepare(b0["caption"])
G.load_next(b0["image"], b0["image_ori"]["faces"], d0["posterior_eps"])
G.load_step(ids, mp, d0["t"], d0["noise"], b0["image_ori"]["ids"])
G.capture()
def rel(a, b): return ((a - b).norm() / b.norm()).item()
def pre(b, d):
    G.load_next(b["image"], b["image_ori"]["faces"], d["posterior_eps"]); G.prefetch(); torch.cuda.synchronize()
    return G.z_n.clone(), G.v_n.clone()
z1, v1 = pre(*bs[1]); z2, v2 = pre(*bs[1])
print("G_pre twice: z", rel(z1, z2), "v", rel(v1, v2))
# eager front end
G.load_next(bs[1][0]["image"], bs[1][0]["image_ori"]["faces"], bs[1][1]["posterior_eps"]); G._front_end(); torch.cuda.synchronize()
print("eager vs G_pre: z", rel(G.z_n, z1), "v", rel(G.v_n, v1))
# inside G_pipe
pre(*bs[0])
G.load_next(bs[1][0]["image"], bs[1][0]["image_ori"]["faces"], bs[1][1]["posterior_eps"]); G.step(lookahead=True); torch.cuda.synchronize()
print("G_pipe front end vs G_pre: z", rel(G.z_n, z1), "v", rel(G.v_n, v1))
G.load_next(bs[1][0]["image"], bs[1][0]["image_ori"]["faces"], bs[1][1]["posterior_eps"]); G.step(lookahead=True); torch.cuda.synchronize()
print("G_pipe again: z", rel(G.z_n, z1), "v", rel(G.v_n, v1))
# eager pipe body
G.load_next(bs[1][0]["image"], bs[1][0]["image_ori"]["faces"], bs[1][1]["posterior_eps"]); G._body_pipe(); torch.cuda.synchronize()
print("eager pipe body: z", rel(G.z_n, z1), "v", rel(G.v_n, v1))
with ops.lane(2):
    zz, _ = eng.encode_first_stage(G.image_n, G.peps_n)
torch.cuda.synchronize()
print("VAE alone lane2: z", rel(zz, z1))
zz0, _ = eng.encode_first_stage(G.image_n, G.peps_n)
torch.cuda.synchronize()
print("VAE alone lane0: z", rel(zz0, z1))
