"""CUDA-graph predictor: the whole hot path (tokenizer -> ViT encoder -> prompt decoder) captured once for
fixed shapes and replayed per cloud.  Inputs may be host (pinned) or device tensors; the H2D copies are
enqueued on the same stream ahead of the replay.  Public API: ``PointCloudSAM.make_predictor``."""
from __future__ import annotations

import torch

from . import engine, native as nv, ops


class GraphPredictor:
    def __init__(self, model, B: int, N: int, P: int, multimask_output: bool = True, use_graph: bool = True,
                 device=None):
        self.model = model
        self.dev = device or next(model.parameters()).device
        self.multimask = multimask_output
        d = self.dev
        self.xyz = torch.zeros((B, N, 3), dtype=torch.float32, device=d)
        self.feats = torch.zeros((B, N, 3), dtype=torch.float32, device=d)
        self.pc = torch.zeros((B, P, 3), dtype=torch.float32, device=d)
        self.pl = torch.zeros((B, P), dtype=torch.int64, device=d)
        self.graph = None
        self.use_graph = use_graph
        self.masks = self.iou = None
        self.launches_per_step = 0
        self.stream = torch.cuda.Stream(device=d)
        # this lane's own out-of-range flag (PositionEmbeddingRandom's ValueError, prompt_encoder.py:44-46): written by the
        # kernels captured in this lane's graph, read back with the result, never shared with other lanes / eager calls
        self.flag = torch.zeros(1, dtype=torch.int32, device=d)
        self.flag_host = torch.zeros(1, dtype=torch.int32).pin_memory()

    def _run(self):
        with engine.flag_scope(range_flag=self.flag):
            return self._run_inner()

    def _run_inner(self):
        import os

        only = os.environ.get("PSAM_PROFILE_STAGE")  # attribution experiments only (tools/stage_attribution.sh)
        if only == "tokenizer":
            from . import engine as _e

            p = _e.run_knn_grouper(self.model.pc_encoder.patch_embed.grouper, self.xyz, self.feats)
            emb = _e.run_patch_encoder(self.model.pc_encoder.patch_embed.patch_encoder, p["features"])
            return emb, emb
        if only == "encoder":
            enc = self.model._encode(self.xyz, self.feats)
            return enc["pc_embeddings"], enc["pc_pe"]
        enc = self.model._encode(self.xyz, self.feats)
        return self.model._decode_unchecked(enc, self.pc, self.pl, None, self.multimask)

    def warmup(self, xyz, feats, pc, pl):
        """Eager passes (pack weights, size the allocator) then capture."""
        with torch.no_grad(), torch.cuda.stream(self.stream):
            self._load(xyz, feats, pc, pl)
            for _ in range(2):
                n0 = nv.LAUNCHES[0]
                self.masks, self.iou = self._run()
                self.launches_per_step = nv.LAUNCHES[0] - n0
            self.stream.synchronize()
            with engine.flag_scope(range_flag=self.flag):
                engine.raise_if_out_of_range(self.dev)
            if self.use_graph:
                self.graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(self.graph, stream=self.stream):
                    self.masks, self.iou = self._run()
        self.stream.synchronize()

    def _load(self, xyz, feats, pc, pl, caller=None):
        """Copies run on the predictor's stream.  Device inputs may have been produced on the caller's stream (GPU
        preprocessing): order this stream behind it.  Pinned host inputs must stay unmodified until the step's result has
        been read (PipelinedPredictor.wait_lane_free)."""
        if caller is not None and caller != self.stream and any(t.is_cuda for t in (xyz, feats, pc, pl)):
            self.stream.wait_stream(caller)
        self.xyz.copy_(xyz, non_blocking=True)
        self.feats.copy_(feats, non_blocking=True)
        self.pc.copy_(pc, non_blocking=True)
        self.pl.copy_(pl, non_blocking=True)

    def __call__(self, xyz, feats, pc, pl, flag_out=None):
        """Enqueue one step on the predictor's stream; returns device tensors (valid after ``check()`` / a stream sync).
        flag_out: pinned int32[1] that receives this step's range flag instead of the lane's own host word."""
        caller = torch.cuda.current_stream(self.dev)
        with torch.no_grad(), torch.cuda.stream(self.stream):
            self._load(xyz, feats, pc, pl, caller)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.masks, self.iou = self._run()
            # the flag travels with the result (4 bytes) and is cleared on-stream for the lane's next step
            (flag_out if flag_out is not None else self.flag_host).copy_(self.flag, non_blocking=True)
            self.flag.zero_()
        return self.masks, self.iou

    def raise_if_flagged(self):
        """Call after the step's completion has been observed (event / stream sync)."""
        if int(self.flag_host[0]) != 0:
            self.flag_host[0] = 0
            raise ValueError("Input coordinates must be normalized to [-1, 1].")

    def check(self):
        """Wait for the enqueued step and raise the reference's ValueError (prompt_encoder.py:44-46) if its coordinates
        or prompts were outside [-1, 1]."""
        self.stream.synchronize()
        self.raise_if_flagged()


class IterativeGraphPredictor:
    """The evaluation loop of the reference (pc_sam.py:90-196 with is_eval=True, as driven by eval_kitti.py:363) for fixed
    shapes [B clouds, M ground-truth masks, N points]: one CUDA graph holds the encoder and all ``model.prompt_iters``
    rounds of batched GT prompt sampling (psam_border_prompt_f32), prompt/mask encoding, two-way decoding and best-mask
    feedback.  The reference synchronises with the host several times per (cloud, mask, iteration); here the only host
    interaction is one flag read after the replay.  Returns the same list of per-iteration dicts as ``forward``."""

    def __init__(self, model, B: int, M: int, N: int, use_graph: bool = True, device=None, throughput_tiles: bool = False):
        self.model = model
        self.dev = device or next(model.parameters()).device
        self.throughput_tiles = throughput_tiles
        d = self.dev
        self.xyz = torch.zeros((B, N, 3), dtype=torch.float32, device=d)
        self.feats = torch.zeros((B, N, 3), dtype=torch.float32, device=d)
        self.gt = torch.zeros((B, M, N), dtype=torch.bool, device=d)
        self.use_graph = use_graph
        self.graph = None
        self.outputs = None
        self.launches_per_step = 0
        self.stream = torch.cuda.Stream(device=d)
        self.flag = torch.zeros(1, dtype=torch.int32, device=d)      # coordinates outside [-1, 1]
        self.sflag = torch.zeros(1, dtype=torch.int32, device=d)     # a ground-truth mask without border

    def _run(self):
        with engine.flag_scope(range_flag=self.flag, sampler=self.sflag):
            return self.model(self.xyz, self.feats, self.gt, is_eval=True)

    def _load(self, xyz, feats, gt, caller=None):
        if caller is not None and caller != self.stream and any(t.is_cuda for t in (xyz, feats, gt)):
            self.stream.wait_stream(caller)
        self.xyz.copy_(xyz, non_blocking=True)
        self.feats.copy_(feats, non_blocking=True)
        self.gt.copy_(gt, non_blocking=True)

    def warmup(self, xyz, feats, gt):
        prev = ops.GEMM_TILE_HINT
        if self.throughput_tiles:
            ops.GEMM_TILE_HINT = 1  # baked into the captured graph
        try:
            with torch.no_grad(), torch.cuda.stream(self.stream):
                self._load(xyz, feats, gt)
                for _ in range(2):
                    n0 = nv.LAUNCHES[0]
                    self.outputs = self._run()  # eager: raises like the reference on bad inputs
                    self.launches_per_step = nv.LAUNCHES[0] - n0
                self.stream.synchronize()
                if self.use_graph:
                    self.graph = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(self.graph, stream=self.stream):
                        self.outputs = self._run()
            self.stream.synchronize()
        finally:
            ops.GEMM_TILE_HINT = prev

    def __call__(self, xyz, feats, gt, check: bool = True):
        caller = torch.cuda.current_stream(self.dev)
        with torch.no_grad(), torch.cuda.stream(self.stream):
            self._load(xyz, feats, gt, caller)
            if self.graph is not None:
                self.graph.replay()
            else:
                self.outputs = self._run()
        if check:
            self.check()
        return self.outputs

    def check(self):
        """One host read for the whole loop: coordinates out of [-1, 1] (ValueError) / masks without a border (RuntimeError)."""
        self.stream.synchronize()
        with engine.flag_scope(range_flag=self.flag, sampler=self.sflag):
            engine.raise_if_out_of_range(self.dev)
            engine.raise_if_sampler_failed(self.dev)


class IterativeGraphPredictorVarlen(IterativeGraphPredictor):
    """PointCloudSAM.forward_varlen as one CUDA graph: static padded buffers xyz / feats [B, N_max, 3], gt [B, M, N_max]
    and lengths [B] (int32, device).  FPS's tie-break block size, the kNN bound and the prompt sampler read the lengths on
    the device, so one capture serves every batch of up to B clouds of at most N_max points each.  Inputs are sequences of
    [N_b, 3], [N_b, 3] and [M, N_b] or [N_b] tensors, as for forward_varlen; the call returns forward_varlen's per-cloud
    lists as views of the graph's outputs, valid until the next call."""

    def __init__(self, model, B: int, M: int, N_max: int, use_graph: bool = True, device=None, throughput_tiles: bool = False):
        super().__init__(model, B, M, N_max, use_graph, device, throughput_tiles)
        self.lengths = torch.zeros(B, dtype=torch.int32, device=self.dev)
        self.sizes = []

    def _run(self):
        with engine.flag_scope(range_flag=self.flag, sampler=self.sflag):
            enc = self.model._encode(self.xyz, self.feats, self.lengths)
            return self.model._eval_loop(enc, self.xyz, self.gt, True, self.lengths)

    def _check(self, coords, features, gt_masks):
        """Host-side refusals, before anything is enqueued."""
        B, M, N_max = self.gt.shape
        if torch.is_tensor(coords) or torch.is_tensor(features):
            raise TypeError("coords and features must be sequences of [N_b, 3] tensors, one per cloud")
        coords, features = list(coords), list(features)
        if len(coords) > B:
            raise ValueError(f"{len(coords)} clouds for a predictor of at most {B}")
        sizes = self.model.varlen_clouds(coords, features)
        if max(sizes) > N_max:
            raise ValueError(f"cloud {sizes.index(max(sizes))} has {max(sizes)} points, more than the predictor's {N_max}")
        if any(f.shape[1] != self.feats.shape[2] for f in features):
            raise ValueError(f"features must be [N_b, {self.feats.shape[2]}]")
        gts = self.model._varlen_gt(gt_masks, sizes)
        if gts[0].shape[0] != M:
            raise ValueError(f"ground truth has {gts[0].shape[0]} masks per cloud, the predictor {M}")
        return coords, features, gts, sizes

    def _load(self, coords, features, gt_masks, caller=None):
        """Cloud b goes to rows 0 .. N_b - 1 of slot b and the rest of the slot is zeroed; slots past the given clouds get
        a copy of the last one (a zero-length cloud would have no border to sample), and their outputs are not returned."""
        coords, features, gts, sizes = self._check(coords, features, gt_masks)
        if caller is not None and caller != self.stream and any(t.is_cuda for t in (*coords, *features, *gts)):
            self.stream.wait_stream(caller)
        slots = [min(b, len(sizes) - 1) for b in range(self.gt.shape[0])]
        self.xyz.zero_()
        self.feats.zero_()
        self.gt.zero_()
        for b, s in enumerate(slots):
            n = sizes[s]
            self.xyz[b, :n].copy_(coords[s], non_blocking=True)
            self.feats[b, :n].copy_(features[s], non_blocking=True)
            self.gt[b, :, :n].copy_(gts[s], non_blocking=True)
        # a fresh pinned tensor per call: a copy still pending from the previous call is never overwritten
        host = torch.tensor([sizes[s] for s in slots], dtype=torch.int32).pin_memory()
        self.lengths.copy_(host, non_blocking=True)
        self.sizes = sizes

    def __call__(self, coords, features, gt_masks, check: bool = True):
        outputs = super().__call__(coords, features, gt_masks, check)
        return self.model._split_varlen(outputs, self.sizes, self.gt.shape[1])


class PipelinedPredictor:
    """Serving front-end: `depth` independent GraphPredictors (own stream, own CUDA graph, own static buffers,
    shared weights) used round-robin, so consecutive clouds overlap on the GPU - cloud i+1's latency-bound FPS /
    small kernels fill the SMs that cloud i's tile-starved GEMMs leave idle.  Each submit() returns a ticket;
    result(ticket) waits for that cloud only."""

    def __init__(self, model, B: int, N: int, P: int, depth: int = 3, multimask_output: bool = True, use_graph: bool = True):
        self.lanes = [GraphPredictor(model, B, N, P, multimask_output, use_graph) for _ in range(depth)]
        self.depth = depth
        self.slots = depth
        self.events = [torch.cuda.Event() for _ in range(depth)]
        self.count = 0
        self.host_out = None
        import os

        self.throughput_tiles = os.environ.get("PSAM_THROUGHPUT_TILES", "1") != "0"
        self.ln_fold = depth >= 8 and self.throughput_tiles  # LayerNorm-free ViT blocks in the captured graphs (engine.BLOCK_LN_POLICY)

    def warmup(self, xyz, feats, pc, pl):
        from . import ops

        prev = ops.GEMM_TILE_HINT
        if self.depth > 1 and self.throughput_tiles:
            ops.GEMM_TILE_HINT = 1  # baked into the captured graphs
        try:
            # LayerNorm-free ViT blocks only when enough clouds are in flight to hide the 16-CTA proj / fc2 launches they need
            with engine.block_ln_fold(self.ln_fold):
                for lane in self.lanes:
                    lane.warmup(xyz, feats, pc, pl)
        finally:
            ops.GEMM_TILE_HINT = prev

    @property
    def launches_per_step(self):
        return self.lanes[0].launches_per_step

    def enable_host_results(self, C: int):
        """Pinned host buffers for the D2H of (mask logits, iou).  TWO result slots per lane: the host may submit a lane's next
        cloud before it has consumed the previous result, so a lane never idles while the host wakes up and launches (the
        end-to-end rate used to trail the device-resident rate by ~4 %)."""
        B, N = self.lanes[0].xyz.shape[:2]
        self.slots = 2 * self.depth
        self.host_out = [(torch.empty((B, C, N), dtype=torch.float32).pin_memory(),
                          torch.empty((B, C), dtype=torch.float32).pin_memory()) for _ in range(self.slots)]
        self.host_flags = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(self.slots)]
        self.events = [torch.cuda.Event() for _ in range(self.slots)]

    def submit(self, xyz, feats, pc, pl, to_host: bool = False) -> int:
        """Ticket t runs on lane t % depth; its host result (to_host) lands in slot t % slots."""
        i = self.count % self.depth
        k = self.count % self.slots
        lane = self.lanes[i]
        masks, iou = lane(xyz, feats, pc, pl, flag_out=self.host_flags[k] if self.host_out is not None else None)
        with torch.cuda.stream(lane.stream):
            if to_host:
                self.host_out[k][0].copy_(masks, non_blocking=True)
                self.host_out[k][1].copy_(iou, non_blocking=True)
            self.events[k].record()
        self.count += 1
        return self.count - 1

    def _raise_if_flagged(self, ticket: int):
        if self.host_out is None:
            return self.lanes[ticket % self.depth].raise_if_flagged()
        f = self.host_flags[ticket % self.slots]
        if int(f[0]) != 0:
            f[0] = 0
            raise ValueError("Input coordinates must be normalized to [-1, 1].")

    def result(self, ticket: int, to_host: bool = False):
        """Wait for that cloud only; raises ValueError for THIS ticket if its coordinates / prompts were outside [-1, 1]
        (the reference raises inside PositionEmbeddingRandom.forward, prompt_encoder.py:44-46).  Device results (to_host
        False) are valid until the lane's next submit; host results until `slots` further submits."""
        self.events[ticket % self.slots].synchronize()
        self._raise_if_flagged(ticket)
        i = ticket % self.depth
        return self.host_out[ticket % self.slots] if to_host else (self.lanes[i].masks, self.lanes[i].iou)

    def wait_lane_free(self, ticket: int):
        """Block until the result slot that `ticket` will use has been produced by its previous owner (ticket - slots): after
        this returns the host may read that result and then reuse the slot."""
        if ticket >= self.slots:
            self.events[ticket % self.slots].synchronize()

    def synchronize(self):
        for lane in self.lanes:
            lane.stream.synchronize()
