"""CUDA-graph executor of the CelebBasis training step with a one-deep software pipeline.

The step has a frozen, no-grad front end (VAE encode + posterior sample, CosFace R100 on the face crops:
ddpm.py:702-759, meta_net.py:329-346) whose result does not depend on the weights being trained, and the trainable chain
(celeb-basis MLP -> CLIP text -> UNet -> loss -> backward -> (W, b) gradients).  The front end of batch i+1 therefore runs
WHILE batch i trains: its throughput-bound 512^2 convolutions fill the SMs that the latency-bound chain of small UNet /
CLIP launches leaves idle.  Every step still does all of its work exactly once (K steps = K front ends + K chains); the
pipeline only changes when the front end of a batch is executed.

The same executor runs the Textual Inversion step (train_step.TextualInversionStep, n_chunks=0): its front end is the
VAE encode alone, and no face buffers exist.

Three graphs over static buffers (torch is buffers / streams / graph capture only):

  G_pre   front end of the batch in the `next` input slot -> (z_next, v_next)
  G_main  promote next->cur; chain on (z_cur, v_cur)                                   (no look-ahead batch)
  G_pipe  promote next->cur; chain on (z_cur, v_cur)  ||  front end of the new `next` batch  (steady state)

The chain runs on a high-priority stream (its many small kernels should never queue behind a wave of VAE CTAs); the
front end runs with ops.lane(1/2) workspaces, so its split-K and GroupNorm launches never share a workspace with the
chain's concurrent ones.
"""
import torch

from . import ops


class StepGraphs:
    def __init__(self, eng, B=1, T=77, n_chunks=2, image_hw=512):
        self.eng = eng
        dev = eng.dev
        self.B, self.T, self.n_chunks = B, T, n_chunks
        lat = image_hw // 8
        f32 = dict(dtype=torch.float32, device=dev)
        faces = n_chunks > 0        # n_chunks = 0: a step without face crops (Textual Inversion)
        # `next` slot: raw inputs of the batch whose front end runs next
        self.image_n = torch.zeros(B, image_hw, image_hw, 3, **f32)
        self.faces_n = torch.zeros(B, image_hw, image_hw, 3 * n_chunks, **f32) if faces else None
        self.peps_n = torch.zeros(B, 4, lat, lat, **f32)
        self.z_n = torch.zeros(B, 4, lat, lat, **f32)
        self.v_n = torch.zeros(n_chunks * B, 512, **f32) if faces else None
        # `cur` slot: what the chain consumes
        self.z = torch.zeros(B, 4, lat, lat, **f32)
        self.v = torch.zeros(n_chunks * B, 512, **f32) if faces else None
        self.ids = torch.zeros(B, T, dtype=torch.int64, device=dev)
        self.map = torch.zeros(B, T, dtype=torch.int32, device=dev)
        self.t = torch.zeros(B, dtype=torch.int64, device=dev)
        self.noise = torch.zeros(B, 4, lat, lat, **f32)
        self.ids_person = torch.zeros(B, n_chunks, dtype=torch.int64, device=dev) if faces else None
        self.loss = None
        self.outs = {}              # per graph: (loss tensor, eng.last of that capture) -- static addresses per graph
        self.g_pre = self.g_main = self.g_pipe = None
        self.next_token = None      # identity of the batch whose front-end result sits in (z_n, v_n)
        self.launches = {}
        self._hi = torch.cuda.Stream(device=dev, priority=-1)     # G_pipe: the chain
        self._lo = torch.cuda.Stream(device=dev)                  # G_pipe: the next batch's front end

    # ---- input staging (host or device sources; pinned host memory makes the copies asynchronous) -----------------
    def load_next(self, image, faces, posterior_eps):
        self.image_n.copy_(image, non_blocking=True)
        if self.faces_n is not None:
            self.faces_n.copy_(faces, non_blocking=True)
        self.peps_n.copy_(posterior_eps, non_blocking=True)

    def load_step(self, ids, map_, t, noise, ids_person=None):
        self.ids.copy_(ids, non_blocking=True)
        self.map.copy_(map_ if torch.is_tensor(map_) else torch.from_numpy(map_), non_blocking=True)
        self.t.copy_(t, non_blocking=True)
        self.noise.copy_(noise, non_blocking=True)
        if self.ids_person is not None:
            self.ids_person.copy_(ids_person, non_blocking=True)

    # ---- the three bodies ------------------------------------------------------------------------------------------
    def _front_end(self):
        self.eng.stage_prefetch(self.image_n, self.faces_n, self.n_chunks, self.peps_n, z_out=self.z_n, v_out=self.v_n)

    def _promote(self):
        self.z.copy_(self.z_n)
        if self.v is not None:
            self.v.copy_(self.v_n)

    def _chain(self):
        self.loss = self.eng.stage_main(self.z, self.v, self.ids_person, self.ids, self.map, self.t, self.noise)
        self._last = dict(self.eng.last)

    def _body_main(self):
        self._promote()
        self._chain()

    def _body_pipe(self):
        self._promote()
        main = torch.cuda.current_stream()
        hi, lo = self._hi, self._lo
        fork = torch.cuda.Event()
        fork.record(main)
        hi.wait_event(fork)
        lo.wait_event(fork)
        with torch.cuda.stream(lo):
            self._front_end()
            j_lo = torch.cuda.Event()
            j_lo.record(lo)
        with torch.cuda.stream(hi):
            self._chain()
            j_hi = torch.cuda.Event()
            j_hi.record(hi)
        main.wait_event(j_lo)
        main.wait_event(j_hi)

    # ---- capture ---------------------------------------------------------------------------------------------------
    def capture(self):
        """Eager warm-up (runs the per-shape GEMM autotuner un-captured, builds every lazily created buffer), then captures
        the three graphs.  Inputs must have been staged with load_next / load_step."""
        from . import lib
        eng = self.eng
        state0 = [x.clone() for x in eng.ema_state()]       # the warm-up steps move the EMA state
        for _ in range(2):
            self._front_end()
            self._body_main()
        self._body_pipe()
        torch.cuda.synchronize()
        pool = None
        self.gemm_record = []       # (desc bytes, flops) of one whole step (pre + main): pointers into the graphs' pool
        for name, body in (("pre", self._front_end), ("main", self._body_main), ("pipe", self._body_pipe)):
            n0 = lib.launch_count()
            ops.GEMM_RECORD = [] if name != "pipe" else None
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, pool=pool):      # the graphs never run concurrently: one shared memory pool
                body()
            pool = g.pool()
            setattr(self, "g_" + name, g)
            self.launches[name] = lib.launch_count() - n0
            if ops.GEMM_RECORD is not None:
                self.gemm_record += ops.GEMM_RECORD
                ops.GEMM_RECORD = None
            if name != "pre":
                self.outs[name] = (self.loss, self._last)
        torch.cuda.synchronize()
        for x, x0 in zip(eng.ema_state(), state0):
            x.copy_(x0)
        return self

    # ---- stepping --------------------------------------------------------------------------------------------------
    def prefetch(self, token=None):
        """Front end of the batch staged in the `next` slot (prologue of the pipeline, or a step without look-ahead)."""
        self.g_pre.replay()
        self.next_token = token

    def step(self, lookahead=False, token=None):
        """Chain on the batch whose front end was produced last (by prefetch() or by the previous step(lookahead=True));
        with lookahead=True the front end of the batch now staged in the `next` slot runs concurrently."""
        name = "pipe" if lookahead else "main"
        getattr(self, "g_" + name).replay()
        self.next_token = token if lookahead else None
        self.loss, self._last = self.outs[name]
        self.eng.last = self._last
        return self.loss
