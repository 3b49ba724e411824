"""Multi-GPU drivers for the per-layer eval loop: one process per GPU, torch.distributed (NCCL on GPUs,
gloo for the CPU tests).

The reference has no distributed backend: cross-GPU movement is `tensor.to(device)` between layer
groups inside one process (opt.py:413-426, llama.py:370-413; SURVEY section 2 #17-18).  The path shards
two ways (SURVEY section 8e):

  * data parallel over samples (`dp_eval`): the eval loop's samples are independent (opt.py:262-264),
    the 2-bit model fits one 80 GB H100 several times over, so every rank holds the packed weights and
    evaluates samples rank, rank+G, ...; the only collective is one all-reduce of (sum NLL, tokens).
  * layer pipeline (`pp_eval`), for models that do not fit one GPU: contiguous layer ranges per rank
    exactly as opt.py:424-426 (or --layers-dist, llama.py:400-413), micro-batch = one sample, hidden
    states (1,S,H) fp16 sent to the next stage with isend/irecv (ncclSend/ncclRecv over NVLink) on one
    communicator per link, receives posted one sample ahead and sends double-buffered so transfers overlap
    the layers; each stage's body is one CUDA-graph replay per sample (`PipelineStage`).
"""
import os

import torch
import torch.distributed as dist

from . import evalloop


def init_distributed(backend=None, device=None):
    """Initialise from the torchrun environment (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_ADDR / MASTER_PORT)."""
    if dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if world == 1:
        return 0, 1
    if backend is None:
        backend = 'nccl' if torch.cuda.is_available() else 'gloo'
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1')
    os.environ.setdefault('MASTER_PORT', '29500')
    kw = {}
    if backend == 'nccl':
        local = int(os.environ.get('LOCAL_RANK', rank))
        torch.cuda.set_device(local)
        kw['device_id'] = torch.device('cuda', local)
    dist.init_process_group(backend=backend, rank=rank, world_size=world, **kw)
    return rank, world


def _allreduce_pair(nll, count):
    t = torch.stack([nll.float(), count.float()])
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t[0], t[1]


@torch.no_grad()
def dp_eval(model, arch, testenc, dev, verbose=False):
    """Data-parallel perplexity: samples round-robin over ranks, one all-reduce at the end."""
    ids = testenc.input_ids if hasattr(testenc, 'input_ids') else testenc
    nsamples = ids.numel() // model.seqlen
    rank, world = (dist.get_rank(), dist.get_world_size()) if dist.is_initialized() else (0, 1)
    mine = list(range(rank, nsamples, world))
    return evalloop.eval_ppl(model, arch, ids, dev, sample_ids=mine, verbose=verbose and rank == 0,
                             reduce_fn=_allreduce_pair if world > 1 else None)


def stage_ranges(nlayers, world, layers_dist=None):
    if layers_dist:
        from .llama import parse_layers_dist
        return parse_layers_dist(layers_dist, nlayers)
    from .opt import layer_placement
    return layer_placement(nlayers, world)


def place_stage(model, arch, lo, hi, dev, first, last):
    """Move only what this pipeline stage needs to `dev`."""
    layers = arch.layers(model)
    for i in range(lo, hi):
        layers[i].to(dev)
    for mod in arch.pre(model):        # every stage derives the layer kwargs (positions / rotary) locally
        mod.to(dev)
    if last:
        for mod in arch.post(model):
            mod.to(dev)
        arch.head(model).to(dev)


_pair_groups = {}


def pair_groups():
    """One process group per adjacent stage pair (r, r+1).  Point-to-point operations on the default group are serialised
    with every other operation on it (NCCL warns about exactly that); with a communicator per link a stage's receive from
    r-1, its send to r+1 and the next receive run independently of each other and of the final all-reduce."""
    world = dist.get_world_size()
    key = (world, dist.get_backend())
    if key not in _pair_groups:
        _pair_groups[key] = [dist.new_group([r, r + 1]) for r in range(world - 1)]      # same order on every rank
    return _pair_groups[key]


class PipelineStage:
    """One rank's contiguous layer range (opt.py:424-426) as a pipeline stage over fixed-length samples.

    * the layer kwargs (mask / positions / rotary tables) are derived ONCE from an example batch -- they are the same for
      every sample of that length -- instead of re-running the embedding front end on every stage for every sample;
    * the stage body (its decoder layers; on the last stage also final norm -> lm_head -> loss) is captured in one CUDA
      graph on CUDA devices and replayed per sample (eager on CPU: the gloo tests);
    * hidden states travel over per-link process groups; the receive of sample j+1 is posted before sample j is computed
      and sends are double-buffered, so transfers overlap the layers.
    """

    def __init__(self, model, arch, lo, hi, dev, example_batch, graph=None):
        self.model, self.arch, self.dev = model, arch, torch.device(dev)
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.first, self.last = self.rank == 0, self.rank == self.world - 1
        self.layers = [arch.layers(model)[i] for i in range(lo, hi)]
        self.groups = pair_groups()
        self.seqlen = example_batch.shape[1]
        with torch.no_grad():
            h0, self.kw = evalloop.layer_inputs(model, arch, example_batch.to(self.dev))
        self.h_in = torch.zeros_like(h0)
        self.labels = example_batch.to(self.dev).clone()
        self.recv_bufs = [torch.empty_like(h0) for _ in range(2)]
        self.send_bufs = [torch.empty_like(h0) for _ in range(2)]
        self.graph = None
        use_graph = self.dev.type == 'cuda' if graph is None else graph
        if use_graph:
            side = torch.cuda.Stream(device=self.dev)
            side.wait_stream(torch.cuda.current_stream(self.dev))
            with torch.no_grad(), torch.cuda.stream(side):
                for _ in range(2):                          # lazy set-up (descriptors, workspaces) outside the graph
                    self._body()
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=side, capture_error_mode='thread_local'):
                    self.out = self._body()
            torch.cuda.current_stream(self.dev).wait_stream(side)

    def _body(self):
        h = evalloop.run_layers(self.model, self.arch, self.layers, self.h_in, self.kw)
        if self.last:
            return evalloop.sample_logits_nll(self.model, self.arch, h, self.labels, self.model.seqlen)
        return h

    def _compute(self):
        if self.graph is not None:
            self.graph.replay()
            return self.out
        return self._body()

    @torch.no_grad()
    def run(self, batches):
        """All samples of `batches` (an indexable of (1, S) id tensors, host or device) through this stage.  Returns the summed
        NLL on the last stage (0 elsewhere)."""
        n = len(batches)
        nll = torch.zeros((), dtype=torch.float32, device=self.dev)
        recv = [None, None]
        sends = [None, None]
        g_in = self.groups[self.rank - 1] if not self.first else None
        g_out = self.groups[self.rank] if not self.last else None
        if not self.first and n:
            recv[0] = dist.irecv(self.recv_bufs[0], src=self.rank - 1, group=g_in)
        for j in range(n):
            if self.first:
                h0, _ = evalloop.layer_inputs(self.model, self.arch, batches[j].to(self.dev, non_blocking=True))
                self.h_in.copy_(h0)
            else:
                if j + 1 < n:                                 # next receive in flight while this sample is computed
                    recv[(j + 1) & 1] = dist.irecv(self.recv_bufs[(j + 1) & 1], src=self.rank - 1, group=g_in)
                recv[j & 1].wait()
                self.h_in.copy_(self.recv_bufs[j & 1])
            if self.last:
                self.labels.copy_(batches[j].to(self.dev, non_blocking=True))
            out = self._compute()
            if self.last:
                nll += out
            else:
                if sends[j & 1] is not None:
                    sends[j & 1].wait()                       # the buffer's previous send (sample j-2) has left
                self.send_bufs[j & 1].copy_(out)
                sends[j & 1] = dist.isend(self.send_bufs[j & 1], dst=self.rank + 1, group=g_out)
        for r in sends:
            if r is not None:
                r.wait()
        return nll


@torch.no_grad()
def pp_eval(model, arch, testenc, dev, layers_dist=None, verbose=False, graph=None):
    """Layer-pipelined perplexity over all ranks of the default process group (reference placement rule opt.py:424-426 /
    --layers-dist llama.py:400-413; NCCL send/recv between neighbours instead of `.to(device)` hops)."""
    ids = testenc.input_ids if hasattr(testenc, 'input_ids') else testenc
    seqlen = model.seqlen
    nsamples = ids.numel() // seqlen
    rank, world = dist.get_rank(), dist.get_world_size()
    layers = arch.layers(model)
    lo, hi = stage_ranges(len(layers), world, layers_dist)[rank]
    first, last = rank == 0, rank == world - 1
    place_stage(model, arch, lo, hi, dev, first, last)
    use_cache = model.config.use_cache
    model.config.use_cache = False
    batches = [ids[:, j * seqlen:(j + 1) * seqlen] for j in range(nsamples)]
    nll = torch.zeros((), dtype=torch.float32, device=dev)
    if nsamples:
        stage = PipelineStage(model, arch, lo, hi, dev, batches[0], graph=graph)
        nll = stage.run(batches)
    count = torch.tensor(float(nsamples * seqlen), device=dev)
    t = torch.stack([nll, count]) if last else torch.zeros(2, device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)         # only the last stage contributes
    ppl = torch.exp(t[0] / t[1]).item()
    if verbose and rank == 0:
        print(ppl)
    model.config.use_cache = use_cache
    return ppl


class PipelinedDecoder:
    """Token-by-token decode with a KV cache across a layer pipeline: the reference's `benchmark()` on a model placed by
    `opt_multigpu` / `llama_multigpu` (opt.py:384-482, llama.py:361-471), one process per GPU.

    Every rank owns one `decode.GraphDecoder` stage (its contiguous layer range, the KV cache of those layers, one CUDA graph
    on CUDA devices); the (batch, 1, hidden) fp16 hidden state of the token travels over the per-link communicators of
    `pair_groups()`.  The token ids are given on every rank (the benchmark is teacher-forced, opt.py:461-470), so nothing
    flows back from the last stage and stage r can start token i+1 while stage r+1 works on token i."""

    def __init__(self, model, arch, dev, max_len=256, batch=1, layers_dist=None, graph=None, ops=None):
        from .decode import GraphDecoder
        self.rank, self.world = dist.get_rank(), dist.get_world_size()
        self.first, self.last = self.rank == 0, self.rank == self.world - 1
        self.dev = torch.device(dev)
        lo, hi = stage_ranges(len(arch.layers(model)), self.world, layers_dist)[self.rank]
        self.groups = pair_groups() if self.world > 1 else []
        self.dec = GraphDecoder(model, max_len=max_len, batch=batch, ops=ops, layer_range=(lo, hi), first=self.first, last=self.last)
        if self.dev.type == 'cuda' if graph is None else graph:
            self.dec.capture()

    def reset(self):
        self.dec.reset()

    @torch.no_grad()
    def step(self, tokens):
        """tokens (batch,) on every rank -> logits (batch, vocab) on the last rank, None elsewhere."""
        if not self.first:
            dist.recv(self.dec.h_in, src=self.rank - 1, group=self.groups[self.rank - 1])
        out = self.dec.step(tokens.to(self.dev))
        if not self.last:
            dist.send(self.dec.h_out, dst=self.rank + 1, group=self.groups[self.rank])
        return out if self.last else None


@torch.no_grad()
def pp_decode_benchmark(model, arch, input_ids, dev, max_len=None, check=False, layers_dist=None, graph=None):
    """`benchmark()` (opt.py:431-482) over the pipeline: feeds input_ids (1, T) token by token.  Returns a dict, the same on
    every rank: `latency_s` = median seconds per token with all ranks synchronised around every token (what a generation loop
    would see), `pipelined_s` = seconds per token of the free-running teacher-forced feed (stages overlapped across tokens), and
    `ppl` of the fed sequence with check (computed on the last rank, as opt.py:469-475 does on the last GPU)."""
    import time

    import torch.nn.functional as F
    dev = torch.device(dev)
    ids = input_ids.reshape(-1).to(dev)
    T = int(ids.numel())
    pd = PipelinedDecoder(model, arch, dev, max_len=max_len or T, batch=1, layers_dist=layers_dist, graph=graph)
    sync = torch.cuda.synchronize if dev.type == 'cuda' else (lambda: None)
    times, tot = [], torch.zeros((), dtype=torch.float32, device=dev)
    for i in range(T):
        sync()
        dist.barrier()
        t0 = time.perf_counter()
        logits = pd.step(ids[i:i + 1])
        sync()
        dist.barrier()
        times.append(time.perf_counter() - t0)
        if check and pd.last and i != T - 1:
            tot += F.cross_entropy(logits.float(), ids[i + 1:i + 2])
    pd.reset()
    sync()
    dist.barrier()
    t0 = time.perf_counter()
    for i in range(T):
        pd.step(ids[i:i + 1])
    sync()
    dist.barrier()
    free = (time.perf_counter() - t0) / T
    stats = torch.tensor([sorted(times)[len(times) // 2], free, float(tot) if pd.last else 0.0], dtype=torch.float64, device=dev)
    dist.all_reduce(stats, op=dist.ReduceOp.MAX)     # times: slowest rank; the NLL sum lives on the last rank only
    ppl = float(torch.exp(stats[2] / (T - 1))) if check and T > 1 else None
    return dict(latency_s=float(stats[0]), pipelined_s=float(stats[1]), ppl=ppl, tokens=T, stages=pd.world)
