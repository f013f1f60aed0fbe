"""Training / evaluation loop with the reference's ``Trainer`` interface (trainer.py:54-285).

    Trainer(model, criterion, optimizer=None, device_ids=[0], device='cuda', dtype=torch.float,
            distributed=False, local_rank=-1, adapt_grad_norm=None, mixup=None, cutmix=None,
            loss_scale=1., grad_clip=-1, print_freq=100)
    .train(loader, average_output=False, chunk_batch=1) / .validate(loader) / .calibrate_bn(loader, num_steps)
        -> dict of meter averages (step, data, loss, prec1, prec5, error1, error5[, grad])

One iteration = zero_grad -> regime update -> H2D -> forward -> loss -> backward -> unscale -> clip ->
optimizer step, as in ``Trainer._step`` (trainer.py:106-177).

B200 path (model converted by engine.convert_b200): inputs stay fp32 NCHW on the device (the stem kernel
does the bf16/NHWC conversion), gradients land in the flat arena, the data-parallel reduction is ONE
NCCL all-reduce of that arena (no DistributedDataParallel wrapper, no per-forward buffer broadcast --
SURVEY.md section 2.3 C1/C2), and the per-tensor unscale / clip loops of the reference
(trainer.py:165-172) are folded into the fused optimizer kernel.

MixUp / CutMix (``mixup`` / ``cutmix``, trainer.py:44-51,119-138): drawn on the host per training chunk by
utils/mixup.py; on the fused B200 path the input relayout and loss kernels do the mixing (see ``_upload_mix``).

Fused training steps loop over the torch.chunks of the batch (``chunk_batch`` N, trainer.py:106-160), the whole batch
being the one-chunk case: each chunk is a fused (captured) step with the loss gradient scaled by 1/N, gradients
accumulate in the arena, the optimizer steps once.  Device-augmented batches split over B*D rows (ops.Aug.row_range).

Augmentation on the device (a loader yielding a utils.augment.DeviceBatch: an AugmentedBatch of data.py
``device_augment`` or a ResizedCropBatch of ``device_resized_crop``): on the fused B200 path the stem relayout kernel
writes the B*D augmented copies from the uint8 data and its draws; every other path trains on the batch's ``apply()``,
the same fp32 batch.  The meters count B*D samples.  Evaluation batches of ``device_scale_crop`` (a ScaleCropBatch:
Resize + CenterCrop) take the same route: with a converted model in eval mode the relayout resamples each image's crop
window and the eval forward runs on it; every other case evaluates the batch's ``apply()``.
"""
import logging
import random
import time

import numpy as np
import torch
import torch.nn as nn
import torch.distributed as dist
from torch.nn.utils import clip_grad_norm_

from .lib import B200Error, MIX_CUTMIX, MIX_MIXUP
from .utils import regularization
from .utils.augment import DeviceBatch, ResizedCropBatch, ScaleCropBatch
from .utils.meters import AverageMeter, accuracy
from .utils.mixup import CutMix, MixUp

_METERS = ('step', 'data', 'loss', 'prec1', 'prec5')


def _flatten_duplicates(inputs, target, batch_first=True, expand_target=True):
    """[B, D, C, H, W] batch-augmentation input -> [(B*D), C, H, W]; targets repeated to match."""
    copies = inputs.size(1)
    if not batch_first:
        inputs = inputs.transpose(0, 1)
    inputs = inputs.flatten(0, 1)
    if expand_target:
        if batch_first:
            target = target.view(-1, 1).expand(-1, copies)
        else:
            target = target.view(1, -1).expand(copies, -1)
        target = target.flatten(0, 1)
    return inputs, target


def _average_duplicates(outputs, target, batch_first=True):
    """Mean of the network outputs over the duplicates of each sample (target is NOT expanded)."""
    bsz = target.size(0)
    if batch_first:
        return outputs.view(bsz, -1, *outputs.shape[1:]).mean(dim=1)
    return outputs.view(-1, bsz, *outputs.shape[1:]).mean(dim=0)


def _mixup(mixup_modules, alpha, batch_size):
    """One module of ``mixup_modules`` draws this chunk's mixing (trainer.py:44-51 of the reference): Python's
    random.sample picks it -- called even for a single candidate, so the Python generator advances as in the
    reference -- then torch.randperm and numpy's beta draw inside ``sample``."""
    for m in mixup_modules:
        m.reset()
    layer = random.sample(mixup_modules, 1)[0]
    layer.sample(alpha, batch_size)
    return layer


def _cuda_prefetch(loader, device, dtype):
    """Yield device-resident batches one step ahead: batch i+1 is copied host->device on a side stream while
    step i computes (the reference issues a blocking copy at the top of every step, trainer.py:116-117).
    The copies land in a ring of three persistent device buffers per (shape, dtype): no caching-allocator traffic per
    step (a fresh 154 MB tensor per batch that is handed across streams made the allocator stall now and then).
    A DeviceBatch's tensors travel together, in the same slot.  The region buffer of a ResizedCropBatch or ScaleCropBatch
    changes size every step: its slots are keyed on a capacity instead, which grows by at least half when a batch does
    not fit."""
    copy_stream = torch.cuda.Stream(device=device)
    ring = {}          # shapes and dtypes -> [[x_buf, y_buf, consumed_event or None, (other device tensors)], ...]
    turn = {}
    capacity = {}      # ring key of ragged batches -> region-buffer bytes

    def stage(inputs, target):
        batch = inputs if isinstance(inputs, DeviceBatch) else None
        host = batch.tensors if batch is not None else (inputs,)
        x, rest = host[0], host[1:]
        x_dtype = x.dtype if x.dtype == torch.uint8 else dtype     # uint8 image batches stay uint8
        ragged = isinstance(batch, (ResizedCropBatch, ScaleCropBatch))
        key = (type(batch), None if ragged else tuple(x.shape), x_dtype, tuple(target.shape), target.dtype,
               tuple((tuple(t.shape), t.dtype) for t in rest))
        shape = tuple(x.shape)
        if ragged:
            cap = capacity.get(key, 0)
            if x.numel() > cap:
                cap = capacity[key] = -(-max(x.numel(), cap * 3 // 2) // (1 << 20)) * (1 << 20)
            shape = (cap,)
        slots = ring.setdefault(key, [])
        k = turn.get(key, 0)
        turn[key] = (k + 1) % 3
        if len(slots) <= k or tuple(slots[k][0].shape) != shape:
            if len(slots) > k and slots[k][2] is not None:
                slots[k][2].synchronize()                 # a grown region buffer replaces one its step has finished with
            new = [torch.empty(shape, device=device, dtype=x_dtype),
                   torch.empty(target.shape, device=device, dtype=target.dtype), None,
                   tuple(torch.empty(t.shape, device=device, dtype=t.dtype) for t in rest)]
            if len(slots) <= k:
                slots.append(new)
            else:
                slots[k] = new
        slot = slots[k]
        with torch.cuda.stream(copy_stream):
            if slot[2] is not None:
                copy_stream.wait_event(slot[2])            # the step that read this slot has been enqueued AND has run
            (slot[0][:x.numel()] if ragged else slot[0]).copy_(x, non_blocking=True)
            slot[1].copy_(target, non_blocking=True)
            for d, t in zip(slot[3], rest):
                d.copy_(t, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(copy_stream)
        return slot, ready, batch

    def hand_over(slot, ready, batch):
        torch.cuda.current_stream(device).wait_event(ready)
        return (slot[0] if batch is None else batch.replace((slot[0],) + slot[3])), slot[1]

    def release(slot):
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))       # everything the consumer enqueued on this batch
        slot[2] = ev

    pending = None
    for inputs, target in loader:
        nxt = stage(inputs, target)
        if pending is not None:
            yield hand_over(*pending)
            release(pending[0])
        pending = nxt
    if pending is not None:
        yield hand_over(*pending)
        release(pending[0])


class Trainer(object):
    def __init__(self, model, criterion, optimizer=None, device_ids=[0], device='cuda', dtype=torch.float,
                 distributed=False, local_rank=-1, adapt_grad_norm=None, mixup=None, cutmix=None,
                 loss_scale=1., grad_clip=-1, print_freq=100):
        self._model = model
        self.criterion = criterion
        self.epoch = 0
        self.training_steps = 0
        self.optimizer = optimizer
        self.device = device
        self.dtype = dtype
        self.distributed = distributed
        self.local_rank = local_rank
        self.print_freq = print_freq
        self.grad_clip = grad_clip
        # input mixing (trainer.py:119-135 of the reference).  With both set the reference builds a CutMix whose alpha
        # is taken from ``mixup`` (mix_val = mixup or cutmix): reproduced as is
        self.mixup = mixup
        self.cutmix = cutmix
        self.last_mix = None                   # the MixUp / CutMix module of the latest training chunk (its draws)
        self._mix_dev, self._mix_ring, self._mix_turn = {}, {}, 0
        self._aug_luts = {}                    # (normalisation, C, device) -> fp32 [C, 256] device LUT of AugmentedBatch
        self.grad_scale = None
        self.loss_scale = loss_scale
        self.adapt_grad_norm = adapt_grad_norm
        self.b200 = getattr(model, '_b200', None)
        self._graphs, self._graph_pool, self._graph_broken, self._graph_static_ok = {}, None, False, None
        self.use_graphs = True
        self.graph_replays = 0                 # bench.py: launches replayed from graphs are not counted by the library
        self.graph_replayed_launches = 0
        self.world_size = dist.get_world_size() if (distributed and dist.is_initialized()) else 1
        self._upstream_t, self._upstream_v = None, None
        self._chunk_w = {}                     # (rows, chunk_batch, device) -> fp32 [k, 3] weights of the chunk meters

        if self.b200 is not None:
            self.model = model
            if optimizer is not None and hasattr(optimizer, 'fold_zero_grad'):
                optimizer.fold_zero_grad(True)     # the fused SGD pass also clears the gradient arena
            if distributed and self.world_size > 1:
                self._broadcast_initial_state()
                self.b200.grad_bucket_hook = Trainer._GradBuckets(self.b200.arena, self.b200.device)
        elif distributed:
            if device_ids and 'cuda' in str(device):
                self.model = nn.parallel.DistributedDataParallel(model, device_ids=device_ids,
                                                                 output_device=device_ids[0])
            else:  # CPU / gloo processes (the reference crashes here: trainer.py:82 with device_ids=None)
                self.model = nn.parallel.DistributedDataParallel(model)
        elif device_ids and len(device_ids) > 1:
            self.model = nn.DataParallel(model, device_ids)
        else:
            self.model = model

    # ------------------------------------------------------------------ data-parallel helpers (B200)
    def _broadcast_initial_state(self):
        """rank 0 -> all: parameters (one flat broadcast) and BN buffers, once (what DDP's ctor does)."""
        arena = self.b200.arena
        dist.broadcast(arena.p32, src=0)
        for buf in self._model.buffers():
            dist.broadcast(buf, src=0)
        arena.sync_shadow()

    def _allreduce_gradients(self, accumulated=False):
        """Sum of the gradient arena over the ranks (the 1/world factor is folded into the SGD kernel).  Normally the
        reduction already ran inside the backward pass -- NCCL all-reduces of arena ranges on a communication stream,
        launched as soon as a range is final and overlapped with the remaining backward kernels (inside the captured
        graph they are graph nodes) -- and nothing is left to do here; the flat all-reduce below serves runs whose
        capture with in-graph all-reduces failed, and fused chunked steps (``accumulated``), whose backward passes keep
        the buckets out: only the sum over the chunks is reduced."""
        if self.b200 is None or self.world_size <= 1 or (self.b200.grad_bucket_hook is not None and not accumulated):
            return
        from . import ops
        g32 = self.b200.arena.g32
        with ops._T('allreduce_nccl', 0, 4 * g32.numel()):
            dist.all_reduce(g32)

    class _GradBuckets(object):
        """engine.Runtime.grad_bucket_hook for data-parallel runs (replaces DistributedDataParallel's bucketed reducer,
        trainer.py:79-82 of the reference)."""

        def __init__(self, arena, device):
            self.g32 = arena.g32
            # host tensors (gloo, CPU tests of the N > 1 logic) have no streams: the reduction is then synchronous
            self.comm = torch.cuda.Stream(device=device) if torch.device(device).type == 'cuda' else None
            self.launched = 0
            self.bytes = 0

        def bucket(self, lo, hi, wg_stream):
            from . import ops
            seg = self.g32[lo:hi]
            self.launched += 1
            self.bytes += 4 * (hi - lo)
            if self.comm is None:
                dist.all_reduce(seg)
                return
            main = torch.cuda.current_stream()
            if ops._TIMING is not None:            # bench.py's per-class timing step: serialised on the main stream
                if wg_stream is not None:
                    main.wait_stream(wg_stream)
                with ops._T('allreduce_nccl', 0, 4 * seg.numel()):
                    dist.all_reduce(seg)
                return
            ev = torch.cuda.Event()
            ev.record(main)
            self.comm.wait_event(ev)
            if wg_stream is not None:              # the weight gradients of this range were produced on the side stream
                ev2 = torch.cuda.Event()
                ev2.record(wg_stream)
                self.comm.wait_event(ev2)
            with torch.cuda.stream(self.comm):
                dist.all_reduce(seg)

        def finish(self):
            if self.comm is not None:
                torch.cuda.current_stream().wait_stream(self.comm)

    # ------------------------------------------------------------------ step capture (B200)
    # The forward + loss + backward of one batch is ~550 kernel launches; issued eagerly from Python they cost
    # about as much host time as the GPU needs to run them.  After two eager steps per (shape, scale) key the
    # sequence is captured once into a CUDA graph and replayed (SURVEY.md section 8(f) row 3).  The optimiser
    # update and the gradient all-reduce stay outside the graph, so learning-rate schedules keep working.
    def _graph_eligible(self):
        if self.b200 is None or not self.use_graphs or self._graph_broken:
            return False
        return self._hooks_static()

    def _hooks_static(self):
        """True when no regularizer needs to run between forward and backward (such hooks can neither be replayed from
        a graph nor wrapped around the fused forward+loss+backward call)."""
        if self._graph_static_ok is None:
            ok = True    # dropout is fine: the mask comes from torch's graph-safe CUDA generator (philox offsets advance per replay)
            opt = self.optimizer
            for o in getattr(opt, 'optim_regime_list', [opt]):
                reg = getattr(o, 'regularizer', None)
                for r in getattr(reg, 'regularization_list', []):
                    if type(r).pre_forward is not regularization.Regularizer.pre_forward or \
                            type(r).pre_backward is not regularization.Regularizer.pre_backward:
                        ok = False
            self._graph_static_ok = ok
        return self._graph_static_ok

    def graphed_forward_backward(self, inputs, target, mix=None, aug=None, chunks=1):
        """Forward + criterion + backward of one device-resident batch through a captured CUDA graph.
        Returns (logits, loss, stats) -- detached device tensors; stats = fp32[3] {loss, top-1 %, top-5 %} when the fused
        loss kernel computed them, else None -- or None when this call has to run eagerly (warm-up steps of
        a new shape, unsupported configuration).  Gradients land in the arena exactly as in the eager path.
        ``mix`` (ops.Mix, from _upload_mix): the step mixes its input; the graph reads the permutation, lambda and box
        from their persistent device buffers, so every replay uses the values uploaded for that step.
        ``aug`` (ops.Aug or ops.Rrc, from _device_aug): the step augments its uint8 data on the device; the graph reads
        the draw tables from static buffers refreshed like the input, so every replay uses that step's draws.
        ``chunks`` > 1: one chunk of a batch split into that many (fused path only): the loss gradient is scaled by
        1 / chunks, gradients accumulate, and the data-parallel buckets stay out of the graph."""
        if not self._graph_eligible() or not inputs.is_cuda:
            return None
        # loss / gradient scales are NOT part of the key: they reach the kernels through a device scalar; neither are
        # the mixing draws (device buffers) -- only the kind of mixing
        key = (tuple(inputs.shape), inputs.dtype, tuple(target.shape), target.dtype, self._model.training,
               mix.kind if mix is not None else 0,
               aug.key if aug is not None else None, chunks > 1)
        st = self._graphs.get(key)
        if st is None:
            st = self._graphs[key] = {'seen': 0, 'graph': None}
        st['seen'] += 1
        if st['graph'] is None:
            if st['seen'] <= 2:
                return None                       # eager warm-up (library handles, allocator, autotuned state)
            try:
                self._capture(st, inputs, target, mix, aug, chunks)
            except Exception as e:  # noqa: BLE001  -- keep training eagerly if capture is impossible here
                if self.b200.grad_bucket_hook is not None:
                    # NCCL inside the capture is the likely culprit: fall back to ONE flat all-reduce after the graph
                    logging.warning('B200: capture with in-graph all-reduce failed (%s); retrying without overlap', e)
                    self.b200.grad_bucket_hook = None
                    self.b200.arena.zero_grad_force()
                    st['seen'] = 2
                    return None
                logging.warning('B200: CUDA-graph capture failed (%s); continuing with eager launches', e)
                self._graph_broken = True
                self._graphs.clear()
                return None
        st['x'].copy_(inputs, non_blocking=True)
        st['y'].copy_(target, non_blocking=True)
        if aug is not None:
            for dst, src in zip(st['aug'], aug.tables):
                dst.copy_(src, non_blocking=True)
        self._upstream(chunks)                    # refresh the device scalar if a scale changed
        st['graph'].replay()
        self.graph_replays += 1
        self.graph_replayed_launches += st['launches']
        return st['out'].detach(), st['loss'].detach(), st['stats']

    def _capture(self, st, inputs, target, mix=None, aug=None, chunks=1):
        from . import lib, ops
        x_s, y_s = torch.empty_like(inputs), torch.empty_like(target)
        x_s.copy_(inputs)
        y_s.copy_(target)
        aug_s = aug.with_tables(tuple(t.clone() for t in aug.tables)) if aug is not None else None
        if self._graph_pool is None:
            self._graph_pool = torch.cuda.graph_pool_handle()
        graph = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        n0 = lib.launch_count()
        up = self._upstream(chunks)
        eps = self._plain_ce_eps() if self._fused_batch(False, target) else None   # graphed steps never average outputs
        # with NCCL all-reduces inside the capture, ProcessGroupNCCL's watchdog thread polls CUDA events concurrently: the
        # default "global" capture mode would treat that as a capture violation
        mode = 'thread_local' if self.b200.grad_bucket_hook is not None else 'global'
        # capture on a HIGH-priority stream: the kernel nodes inherit it, so when a main-chain kernel (BN backward ->
        # dgrad of the next unit) and a side-stream weight gradient become ready together the block scheduler starts the
        # critical one first and the wgrad CTAs fill in beside the HBM-bound BN kernels that follow
        if getattr(self, '_capture_stream', None) is None:
            self._capture_stream = torch.cuda.Stream(device=x_s.device, priority=-1)
        with torch.cuda.graph(graph, pool=self._graph_pool, stream=self._capture_stream, capture_error_mode=mode):
            stats = None
            if eps is not None:            # the whole step is library calls: nothing of autograd inside the graph
                out, stats = self.b200.train_step(x_s, y_s, eps, up, mix=mix, aug=aug_s, reduce=chunks == 1)
                loss = stats[0]
            else:
                out = self.model(x_s)
                loss = self.criterion(out, y_s)
                torch.autograd.backward(loss, grad_tensors=[up])
        st.update(graph=graph, x=x_s, y=y_s, aug=aug_s.tables if aug_s is not None else None, out=out, loss=loss,
                  stats=stats, launches=lib.launch_count() - n0)

    def release_graphs(self):
        """Drop every captured step (call before tearing the process group down: graphs that captured NCCL all-reduces
        keep the communicator busy and destroy_process_group() can block on them)."""
        self._graphs.clear()
        self._graph_pool = None
        import gc
        gc.collect()
        if torch.cuda.is_available():
            torch.cuda.synchronize()

    def _plain_ce_eps(self):
        """label-smoothing coefficient when the criterion is the reference's plain CrossEntropyLoss (class indices,
        mean reduction, no weights / soft targets / ignore index) -- the case engine.Runtime.train_step fuses;
        None otherwise (generic autograd path)."""
        from .utils.cross_entropy import CrossEntropyLoss
        c = self.criterion
        if type(c) is CrossEntropyLoss and c.weight is None and c.smooth_dist is None and c.reduction == 'mean' \
                and c.ignore_index < 0 and c.from_logits:
            return float(c.smooth_eps or 0.0)
        return None

    def _upstream(self, chunks=1):
        """d(scaled loss)/d(loss) = grad_scale * loss_scale (trainer.py:158-161 of the reference multiplies the loss)
        as a persistent 0-dim device tensor handed to autograd.backward: no per-step scalar kernels, and a captured
        graph reads the current value instead of a baked-in constant.  ``chunks`` > 1: that value divided by chunks in
        fp32, what autograd hands the chunk's loss for the reference's ``loss / chunk_batch`` (trainer.py:146-147)."""
        v = 1.0
        if self.grad_scale is not None:
            v *= float(self.grad_scale)
        if self.loss_scale is not None:
            v *= float(self.loss_scale)
        if chunks > 1:
            v = float(np.float32(v) / np.float32(chunks))
        if self._upstream_t is None:
            self._upstream_t = torch.empty((), device=self.b200.device, dtype=torch.float32)
        if v != self._upstream_v:
            self._upstream_t.fill_(v)
            self._upstream_v = v
        return self._upstream_t

    # ------------------------------------------------------------------ one optimisation step
    def _input_dtype(self):
        return torch.float if self.b200 is not None else self.dtype

    def _grad_norm(self, inputs_batch, target_batch, chunk_batch=1):
        if self.b200 is not None:
            # nn.Module.zero_grad() only drops the views (p.grad = None): the kernels accumulate into the arena itself
            self.b200.arena.zero_grad()
            self.b200.arena.rebind_grads()
        else:
            self.model.zero_grad()
        for inputs, target in zip(inputs_batch.chunk(chunk_batch, dim=0), target_batch.chunk(chunk_batch, dim=0)):
            target = target.to(self.device)
            inputs = inputs.to(self.device, dtype=self._input_dtype())
            loss = self.criterion(self.model(inputs), target)
            if chunk_batch > 1:
                loss = loss / chunk_batch
            loss.backward()
        return clip_grad_norm_(self.model.parameters(), float('inf'))

    def _step(self, inputs_batch, target_batch, training=False, average_output=False, chunk_batch=1):
        """-> (outputs, loss, grad norm or None).  ``loss`` is a float, or -- on the fused B200 path -- the fp32[3] device
        tensor {loss, top-1 %, top-5 %} of the loss kernel, which Trainer.forward reads back asynchronously
        (the reference synchronises three times per step here: trainer.py:153,226-227)."""
        grad = None
        if training:
            self.optimizer.zero_grad()
            self.optimizer.update(self.epoch, self.training_steps)
        fused = training and self._fused_batch(average_output, target_batch)
        if fused:
            output, loss = self._fused_step(inputs_batch, target_batch, chunk_batch)
        elif not training and isinstance(inputs_batch, ScaleCropBatch) and self.b200 is not None \
                and not self.model.training and chunk_batch == 1 and not average_output and 'cuda' in str(self.device):
            # Runtime.forward's eval pass, fed by the relayout of the batch's uint8 regions
            aug, regions = self._device_aug(inputs_batch)
            regions, target = self._to_device(regions, target_batch)
            output = self.b200.run_forward(regions, False, False, aug=aug)[0]
            loss = float(self.criterion(output, target).detach())
            output = output.detach()
        else:
            if isinstance(inputs_batch, DeviceBatch):
                inputs_batch = inputs_batch.apply()     # the same fp32 batch the fused relayout would compute
            outputs, total_loss = [], 0
            for i, (inputs, target, _) in enumerate(self._chunks(inputs_batch, target_batch, chunk_batch, None)):
                is_u8 = inputs.dtype == torch.uint8
                inputs, target = self._to_device(inputs, target)
                mixer = None
                if training and (self.mixup is not None or self.cutmix is not None):
                    mixer = self._draw_mix(inputs.size(0), average_output)
                if training and chunk_batch == 1 and not average_output and mixer is None:
                    replayed = self.graphed_forward_backward(inputs, target)
                    if replayed is not None:
                        outputs.append(replayed[0])
                        total_loss += float(replayed[1])
                        continue
                if mixer is not None:
                    # the reference's fp32 mixing of the batch on its device and the soft target through the criterion
                    if is_u8:
                        raise B200Error('mixup / cutmix of a uint8 batch needs the fused path (plain CrossEntropyLoss, '
                                        'a converted model); normalise the batch to fp32 otherwise')
                    inputs = mixer(inputs.clone() if isinstance(mixer, CutMix) else inputs)   # the caller's batch stays intact
                if training:
                    self.optimizer.pre_forward()
                output = self.model(inputs)
                if average_output:
                    if isinstance(output, (list, tuple)):
                        output = [_average_duplicates(o, target) if o is not None else None for o in output]
                    else:
                        output = _average_duplicates(output, target)
                if mixer is not None:
                    target = mixer.mix_target(target, (output[0] if isinstance(output, (list, tuple)) else output).size(-1))
                loss = self.criterion(output, target)
                if chunk_batch > 1:
                    loss = loss / chunk_batch
                if isinstance(output, (list, tuple)):
                    output = output[0]
                outputs.append(output.detach())
                total_loss += float(loss.detach())

                if training:
                    if i == 0:
                        self.optimizer.pre_backward()
                    if self.b200 is not None and loss.dim() == 0 and loss.dtype == torch.float32:
                        torch.autograd.backward(loss, grad_tensors=[self._upstream()])
                    else:
                        if self.grad_scale is not None:
                            loss = loss * self.grad_scale
                        if self.loss_scale is not None:
                            loss = loss * self.loss_scale
                        loss.backward()
            output, loss = (outputs[0] if len(outputs) == 1 else torch.cat(outputs, dim=0)), total_loss

        if training:
            if self.b200 is not None:
                self._allreduce_gradients(accumulated=fused and chunk_batch > 1)
                self.optimizer.set_grad_unscale(self.loss_scale if self.loss_scale is not None else 1.0,
                                                self.world_size)
                if self.grad_clip > 0:
                    self.optimizer.request_clip(self.grad_clip)
                self.optimizer.step()
                if self.grad_clip > 0:
                    grad = self.optimizer.last_grad_norm
            else:
                if self.loss_scale is not None:
                    for p in self.model.parameters():
                        if p.grad is not None:
                            p.grad.data.div_(self.loss_scale)
                if self.grad_clip > 0:
                    grad = clip_grad_norm_(self.model.parameters(), self.grad_clip)
                self.optimizer.step()
            self.training_steps += 1

        return output, loss, grad

    def _fused_step(self, inputs_batch, target_batch, chunk_batch):
        """-> (logits, fp32[3] statistics) of one training batch on the runtime's fused train_step.  Each torch.chunk of
        the batch -- the whole batch when chunk_batch == 1 -- runs as one fused (captured) step with the loss gradient
        scaled by 1 / chunk_batch; gradients accumulate in the arena (trainer.py:114-147 of the reference).  Several
        chunks' logits and statistics are gathered on the device -- a graph replay overwrites its static outputs."""
        aug = None
        if isinstance(inputs_batch, DeviceBatch):
            aug, inputs_batch = self._device_aug(inputs_batch)
        if chunk_batch > 1:
            from . import ops
            ranges = ops.chunk_rows(target_batch.size(0), chunk_batch)
            chunk_stats = torch.empty((len(ranges), 3), device=self.device, dtype=torch.float32)
        for i, (inputs, target, aug_i) in enumerate(self._chunks(inputs_batch, target_batch, chunk_batch, aug)):
            inputs, target = self._to_device(inputs, target)
            mix = None
            if self.mixup is not None or self.cutmix is not None:
                mix = self._upload_mix(self._draw_mix(inputs.size(0)), inputs)
            self.optimizer.pre_forward()       # static hooks (_hooks_static): this and pre_backward reach no-ops
            replayed = self.graphed_forward_backward(inputs, target, mix, aug_i, chunks=chunk_batch)
            if replayed is not None:
                output, stats = replayed[0], replayed[2]
            else:
                output, stats = self.b200.train_step(inputs, target, self._plain_ce_eps(), self._upstream(chunk_batch),
                                                     mix=mix, aug=aug_i, reduce=chunk_batch == 1)
            if i == 0:
                self.optimizer.pre_backward()
            if chunk_batch == 1:
                return output, stats
            if i == 0:
                chunk_logits = torch.empty((ranges[-1][1], output.shape[1]), device=output.device, dtype=output.dtype)
            chunk_logits[ranges[i][0]:ranges[i][1]].copy_(output)
            chunk_stats[i].copy_(stats)
        return chunk_logits, (chunk_stats * self._chunk_weights(ranges, chunk_batch)).sum(0)

    def _to_device(self, inputs, target):
        """-> (inputs, target) on the device; a converted model's uint8 batches stay uint8 (its relayout normalises)."""
        target = target.to(self.device, non_blocking=True)
        if self.b200 is not None and inputs.dtype == torch.uint8:
            return inputs.to(self.device, non_blocking=True), target
        return inputs.to(self.device, dtype=self._input_dtype(), non_blocking=True), target

    def _fused_training(self, average_output):
        """True when a training step runs as the runtime's fused train_step (plain CrossEntropyLoss, static hooks, a
        converted model on CUDA, no averaged outputs); the targets must also be class indices (_fused_batch)."""
        return self.b200 is not None and not average_output and 'cuda' in str(self.device) and self._hooks_static() \
            and self._plain_ce_eps() is not None

    def _fused_batch(self, average_output, target):
        """True when a training batch with these targets runs as the runtime's fused train_step."""
        return self._fused_training(average_output) and target.dtype == torch.long and target.dim() == 1

    @staticmethod
    def _chunks(inputs_batch, target_batch, chunk_batch, aug):
        """-> (inputs, target, aug) per chunk: torch.chunk of the batch and its targets over the rows, the reference's
        split (trainer.py:114-115).  With device augmentation the B*D rows are split the same way; each chunk's relayout
        reads the images (or regions) that cover its rows and keeps just those rows (ops.Aug.row_range)."""
        if chunk_batch == 1:
            return [(inputs_batch, target_batch, aug)]
        if aug is None:
            return [(x, y, None) for x, y in zip(inputs_batch.chunk(chunk_batch, dim=0),
                                                 target_batch.chunk(chunk_batch, dim=0))]
        from . import ops
        out = []
        for r0, r1 in ops.chunk_rows(target_batch.size(0), chunk_batch):
            a, b0, b1 = aug.row_range(r0, r1)
            out.append((inputs_batch if isinstance(aug, ops.Rrc) else inputs_batch[b0:b1], target_batch[r0:r1], a))
        return out

    def _chunk_weights(self, ranges, chunk_batch):
        """fp32 [k, 3] device weights that combine the chunks' {loss, top-1 %, top-5 %} into the step's meters as the
        reference computes them: the loss is the sum of each chunk's loss / chunk_batch (trainer.py:146-151), the
        accuracies are those of the concatenated outputs, so each chunk counts by its rows."""
        rows = ranges[-1][1]
        key = (rows, chunk_batch, str(self.device))
        w = self._chunk_w.get(key)
        if w is None:
            w = self._chunk_w[key] = torch.tensor([[1.0 / chunk_batch, (r1 - r0) / rows, (r1 - r0) / rows]
                                                   for r0, r1 in ranges], dtype=torch.float32).to(self.device)
        return w

    # ------------------------------------------------------------------ input mixing (MixUp / CutMix)
    def _draw_mix(self, batch_size, average_output=False):
        """This chunk's mixing draws, made on the host in the reference's order (trainer.py:119-131): random.sample,
        torch.randperm, numpy beta (and, for CutMix, the box centre when the batch is mixed).  Returns the module."""
        if average_output:
            # the permutation would run over the B*D duplicated rows while the averaged output and the target have B
            # rows: the reference fails in mix_target here
            raise NotImplementedError('mixup / cutmix with average_output: the mixing permutation covers the B*D '
                                      'duplicated inputs but the averaged outputs and targets have B rows')
        input_mixup = CutMix() if self.cutmix else MixUp()
        # ResNet(mixup=True) intermediate mixing layers are not supported, so the input mixer is the only candidate
        self.last_mix = _mixup([input_mixup], self.mixup or self.cutmix, batch_size)
        return self.last_mix

    _MIX_RING = 4

    def _upload_mix(self, mixer, inputs):
        """-> ops.Mix over persistent device buffers holding this step's permutation and {lambda, r0, r1, c0, c1}.
        One int64 device buffer per batch size: [perm (B) | parameter block (3 words)]; a CUDA graph captured with it
        reads whatever the latest upload wrote.  The host side stages through a small ring of pinned buffers (an event
        guards each slot until its copy has run) and issues ONE non-blocking copy on the current stream, which orders
        it after the previous step's kernels: no host synchronisation per step."""
        from . import ops
        B = inputs.size(0)
        H, W = (inputs.shape[1], inputs.shape[2]) if inputs.dtype == torch.uint8 else (inputs.shape[-2], inputs.shape[-1])
        if isinstance(mixer, CutMix):
            kind, box = MIX_CUTMIX, mixer.draw_box(H, W)     # the reference draws the box when the batch is mixed
        else:
            kind, box = MIX_MIXUP, (0, 0, 0, 0)
        dev = self._mix_dev.get(B)
        if dev is None:
            dev = self._mix_dev[B] = torch.zeros(B + 3, dtype=torch.int64, device=inputs.device)
        ring = self._mix_ring.setdefault(B, [])
        k = self._mix_turn % self._MIX_RING
        self._mix_turn += 1
        if len(ring) <= k:
            ring.append([torch.zeros(B + 3, dtype=torch.int64).pin_memory(), None])
        host, ev = ring[k]
        if ev is not None:
            ev.synchronize()                           # the copy that last read this slot has run (long ago)
        h = host.numpy()
        h[:B] = mixer.mix_index.numpy()
        blk = h[B:].view(np.int32)
        blk[0:1].view(np.float32)[0] = mixer.mix_values.numpy()[0]
        blk[1:5] = box
        dev.copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        ring[k][1] = ev
        return ops.Mix(dev[:B], dev[B:].view(torch.int32), kind)

    # ------------------------------------------------------------------ batch augmentation on the device
    def _device_aug(self, batch):
        """-> (ops.Aug, ops.Rrc or ops.ScaleCropTables over the batch's tables on the device and a persistent device LUT
        of its normalisation -- one per statistics, channel count and device, so that a captured graph keeps reading a
        live tensor --, the uint8 tensor the relayout reads).  Resized-crop tables are validated on the host here: a
        graph replay runs the kernel without passing through ops.input_prep_u8_rrc.  Scale-crop (evaluation) steps are
        not captured; ops.input_prep_u8_scale_crop validates their tables."""
        from . import ops
        spec = batch.spec
        device = torch.device(self.device)
        C = batch.channels if isinstance(batch, (ResizedCropBatch, ScaleCropBatch)) else batch.images.shape[-1]
        key = (tuple(spec.normalize['mean']), tuple(spec.normalize['std']), C, str(device))
        lut = self._aug_luts.get(key)
        if lut is None:
            lut = self._aug_luts[key] = spec.lut(C).to(device)
        if isinstance(batch, ScaleCropBatch):
            sc = ops.ScaleCropTables(batch.index.to(device, non_blocking=True), batch.geom.to(device, non_blocking=True),
                                     lut, spec.size, batch.host + (batch.nbytes,))
            return sc, batch.regions
        if isinstance(batch, ResizedCropBatch):
            ops.check_rrc_tables(batch.host[0], batch.host[1], batch.nbytes, C, spec.duplicates)
            rrc = ops.Rrc(batch.index.to(device, non_blocking=True), batch.draws.to(device, non_blocking=True), lut,
                          spec.duplicates, spec.size, batch.host + (batch.nbytes,))
            return rrc, batch.regions
        params = batch.params.to(device, non_blocking=True).reshape(-1, batch.params.shape[-1])
        # a resize to the images' own size is the identity: that case stays on the kernel without the resample
        out_hw = spec.resize if spec.resize != tuple(batch.images.shape[1:3]) else None
        return ops.Aug(params, lut, spec.duplicates, spec.padding, out_hw), batch.images

    def _check_device_augment(self, training, average_output):
        if average_output:
            raise NotImplementedError('batch augmentation on the device with average_output: the outputs would be '
                                      'averaged over the duplicates; use the [B, D, C, H, W] loader instead')
        if training and (self.mixup is not None or self.cutmix is not None):
            raise NotImplementedError('batch augmentation on the device is not combined with mixup / cutmix')
        if training and self.adapt_grad_norm is not None:
            raise NotImplementedError('batch augmentation on the device with adapt_grad_norm: the per-copy gradient '
                                      'norms need the [B, D, C, H, W] batch; use the host-side loader instead')

    # ------------------------------------------------------------------ epoch loop
    def forward(self, data_loader, num_steps=None, training=False, average_output=False, chunk_batch=1):
        meters = {name: AverageMeter() for name in _METERS}
        if training and self.grad_clip > 0:
            meters['grad'] = AverageMeter()
        batch_first = not ((training and isinstance(self.model, nn.DataParallel)) or chunk_batch > 1)

        def summary():
            res = {name: m.avg for name, m in meters.items()}
            res['error1'] = 100. - res['prec1']
            res['error5'] = 100. - res['prec5']
            return res

        try:
            n_batches = len(data_loader)
        except TypeError:
            n_batches = -1
        tick = time.time()
        batches = _cuda_prefetch(data_loader, self.device, self._input_dtype()) \
            if (self.b200 is not None and (chunk_batch == 1 or (training and self._fused_training(average_output)))) \
            else data_loader
        # lazy meters (B200 fused path): the step's {loss, prec1, prec5} come from the loss kernel as one device
        # tensor; it is copied to pinned host memory asynchronously every step and only awaited when a log line is
        # due, the ring is full or the loop ends -- no host synchronisation inside a step
        pending, ring = [], 8
        pinned = None

        def drain(keep=0):
            while len(pending) > keep:
                slot, ev, n = pending.pop(0)
                ev.synchronize()
                v = pinned[slot]
                meters['loss'].update(float(v[0]), n)
                meters['prec1'].update(float(v[1]), n)
                meters['prec5'].update(float(v[2]), n)

        for i, (inputs, target) in enumerate(batches):
            if isinstance(inputs, DeviceBatch):
                self._check_device_augment(training, average_output)
            duplicates = not isinstance(inputs, DeviceBatch) and inputs.dim() > 4  # B x D x C x H x W
            if training and duplicates and self.adapt_grad_norm is not None and i % self.adapt_grad_norm == 0:
                per_copy = sum(float(self._grad_norm(inputs.select(1, j), target)) for j in range(inputs.size(1)))
                per_copy /= inputs.size(1)
                joint = float(self._grad_norm(*_flatten_duplicates(inputs, target, batch_first)))
                self.grad_scale = per_copy / joint
                logging.info('New loss scale: %s', self.grad_scale)

            meters['data'].update(time.time() - tick)
            if duplicates:
                inputs, target = _flatten_duplicates(inputs, target, batch_first,
                                                     expand_target=not average_output)
            output, loss, grad = self._step(inputs, target, training=training, average_output=average_output,
                                            chunk_batch=chunk_batch)
            n = inputs.rows if isinstance(inputs, DeviceBatch) else inputs.size(0)
            if torch.is_tensor(loss):              # fused statistics: asynchronous read-back
                if pinned is None:
                    pinned = torch.empty((ring, 3), dtype=torch.float32).pin_memory()
                drain(keep=ring - 1)
                slot = i % ring
                pinned[slot].copy_(loss, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record()
                pending.append((slot, ev, n))
                if i % self.print_freq == 0 or i == n_batches - 1:
                    drain()
            else:
                drain()
                target_dev = target.to(output.device)
                prec1, prec5 = accuracy(output, target_dev, topk=(1, 5))
                meters['loss'].update(float(loss), n)
                meters['prec1'].update(float(prec1), n)
                meters['prec5'].update(float(prec5), n)
            if grad is not None:
                meters['grad'].update(float(grad), n)
            meters['step'].update(time.time() - tick)
            tick = time.time()

            if i % self.print_freq == 0 or i == n_batches - 1:
                msg = ('{phase} - Epoch: [{0}][{1}/{2}]\t'
                       'Time {m[step].val:.3f} ({m[step].avg:.3f})\t'
                       'Data {m[data].val:.3f} ({m[data].avg:.3f})\t'
                       'Loss {m[loss].val:.4f} ({m[loss].avg:.4f})\t'
                       'Prec@1 {m[prec1].val:.3f} ({m[prec1].avg:.3f})\t'
                       'Prec@5 {m[prec5].val:.3f} ({m[prec5].avg:.3f})\t').format(
                    self.epoch, i, n_batches, phase='TRAINING' if training else 'EVALUATING', m=meters)
                if 'grad' in meters:
                    msg += 'Grad {m[grad].val:.3f} ({m[grad].avg:.3f})'.format(m=meters)
                logging.info(msg)
            if num_steps is not None and i >= num_steps:  # (sic) the reference runs num_steps+1 iterations
                break
        drain()
        return summary()

    def train(self, data_loader, average_output=False, chunk_batch=1):
        self.model.train()
        return self.forward(data_loader, training=True, average_output=average_output, chunk_batch=chunk_batch)

    def validate(self, data_loader, average_output=False):
        self.model.eval()
        with torch.no_grad():
            return self.forward(data_loader, average_output=average_output, training=False)

    def calibrate_bn(self, data_loader, num_steps=None):
        """Re-estimate BN running statistics as a cumulative average over the loader (momentum=None)."""
        from .models.modules.lp_norm import L1BatchNorm2d
        if any(isinstance(m, L1BatchNorm2d) for m in self.model.modules()):
            raise NotImplementedError('calibrate_bn is not implemented for L1 BatchNorm layers (bn_norm=\'L1\')')
        for m in self.model.modules():
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                m.momentum = None
                m.track_running_stats = True
                m.reset_running_stats()
        self.model.train()
        with torch.no_grad():
            return self.forward(data_loader, num_steps=num_steps, training=False)

    # tensorwatch hooks of the reference (trainer.py:287-337) are observability extras, not part of the path
    def set_watcher(self, filename, port=0):
        return False
