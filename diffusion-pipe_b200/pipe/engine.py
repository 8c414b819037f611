"""PipelineEngine: executes the 1F1B instruction stream over the local stage.

Replaces `deepspeed.initialize(...)` -> PipelineEngine as used by the reference (train.py:623-631, 817-823, 915-918,
181-183; utils/dataset.py:1387-1405; utils/saver.py:59-128).  Semantics restated from deepspeed==0.18.4
runtime/pipe/engine.py as recorded in SURVEY.md section 8a rows E3-E11:

  LoadMicroBatch   first stage: inputs = clone().detach().to(device), requires_grad = is_floating_point;
                   last stage: labels -> device                                                     (E3)
  ForwardPass      local layers in order; last stage loss = loss_fn(outputs, labels)                (E4)
  BackwardPass     last stage (loss / GAS).backward(); else autograd.backward(float outputs, received grads)  (E5)
  Send/Recv*       every tensor of the boundary tuple; grads for every floating-point tensor        (E6)
  ReduceGrads      data-parallel mean of all trainable grads in `communication_data_type`           (E7)
  OptimizerStep    global-norm clip (utils/patches.py:175-246) -> optimizer.step -> zero_grad -> lr_scheduler.step (E8, E9)
  train_batch      returns mean micro-batch loss, averaged over DP and broadcast to every stage      (E10)

Stage links: `DistLink` moves boundary tensors with torch.distributed p2p (gloo on CPU, NCCL on GPUs);
`IpcLink` (pipe/ipc_link.py) is the single-node path — peer copies into pre-registered slots over NVLink with device-side
flags, no NCCL on the boundary.  Selected by `config['stage_link']` ('auto' picks IpcLink on CUDA).
"""
import os
import time

import torch

from . import dist
from .module import PipelineModule
from .schedule import (BackwardInput, BackwardPass, BackwardWeight, ForwardPass, InferenceSchedule, LoadMicroBatch,
                       OptimizerStep, RecvActivation, RecvGrad, ReduceGrads, ReduceTiedGrads, SendActivation, SendGrad,
                       TrainSchedule, ZeroBubbleSchedule)

_DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8,
           torch.bool, torch.float64, torch.complex64]
_DTYPE_ID = {d: i for i, d in enumerate(_DTYPES)}


class DistLink:
    """Boundary transport over torch.distributed point-to-point (same scheme as DeepSpeed: a metadata message when
    shapes are unknown, then one message per tensor)."""

    def __init__(self, engine):
        self.engine = engine
        self.device = engine.device
        self._pending = []
        self.reset()

    def reset(self):
        self._send_meta_done = {}
        self._recv_meta = {}

    def _send(self, t, dst):
        """blocking send for the reference order; isend (completed in flush) when a stage may run ahead of its
        neighbour (zero-bubble order), where two blocking sends could face each other"""
        if self.engine.pipeline_schedule == 'zb':
            self._pending.append((dist.tdist.isend(t, dst), t))
        else:
            dist.send(t, dst)

    def flush(self):
        for w, _t in self._pending:
            w.wait()
        self._pending = []

    def _meta_device(self):
        return self.device if self.device.type == 'cuda' else torch.device('cpu')

    def send_tuple(self, tensors, dst, key):
        meta = [len(tensors)]
        for t in tensors:
            meta += [_DTYPE_ID[t.dtype], t.dim()] + list(t.shape)
        if key not in self._send_meta_done:
            m = torch.tensor([len(meta)] + meta, dtype=torch.int64, device=self._meta_device())
            self._send(m[:1].clone(), dst)
            self._send(m[1:].contiguous(), dst)
            self._send_meta_done[key] = meta
        elif self._send_meta_done[key] != meta:
            # the receiver allocates from the shapes announced once per step: a different tuple would be received into
            # wrongly sized buffers without any error from the transport
            raise RuntimeError('the boundary tuple changed shape or dtype since it was announced to the next stage: call '
                               'engine.reset_activation_shape() before a step whose micro-batches have new shapes '
                               '(train.py:916, train.py:181)')
        for t in tensors:
            self._send(t.contiguous(), dst)

    def recv_tuple(self, src, key):
        if key not in self._recv_meta:
            n = torch.zeros(1, dtype=torch.int64, device=self._meta_device())
            dist.recv(n, src)
            m = torch.zeros(int(n.item()), dtype=torch.int64, device=self._meta_device())
            dist.recv(m, src)
            m = m.tolist()
            specs, pos = [], 1
            for _ in range(m[0]):
                dt, nd = _DTYPES[m[pos]], m[pos + 1]
                specs.append((dt, tuple(m[pos + 2:pos + 2 + nd])))
                pos += 2 + nd
            self._recv_meta[key] = specs
        out = []
        for dt, shape in self._recv_meta[key]:
            t = torch.empty(shape, dtype=dt, device=self.device)
            dist.recv(t, src)
            out.append(t)
        return tuple(out)

    # ---- the engine's four boundary operations ----
    def send_activations(self, outputs, buf, mb, keep=True):
        self.send_tuple(tuple(outputs), self.engine.grid.stage_to_global(self.engine.next_stage), ('act', len(outputs)))

    def recv_activations(self, buf, mb):
        return self.recv_tuple(self.engine.grid.stage_to_global(self.engine.prev_stage), 'act')

    def send_grads(self, grads, buf, mb):
        dst = self.engine.grid.stage_to_global(self.engine.prev_stage)
        for g in grads:
            self._send(g.contiguous(), dst)

    def recv_grads(self, like, buf, mb):
        src = self.engine.grid.stage_to_global(self.engine.next_stage)
        out = []
        for t in like:
            g = torch.empty_like(t, memory_format=torch.contiguous_format)
            dist.recv(g, src)
            out.append(g)
        return out

    def release_grads(self, buf, mb):
        pass        # received tensors are ordinary allocations: nothing to hand back (IpcLink recycles mailbox slots here)

    def release_activations(self, buf, mb):
        pass


class PipelineEngine:
    def __init__(self, model, config, args=None):
        assert isinstance(model, PipelineModule), 'model must be a PipelineModule'
        self.module = model
        self.config = dict(config or {})
        self.grid = model._grid
        self.num_stages = self.grid.pipe_parallel_size
        self.stage_id = self.grid.get_stage_id()
        self.prev_stage = self.stage_id - 1
        self.next_stage = self.stage_id + 1
        self.global_rank = self.grid.global_rank
        self.is_pipe_parallel = self.num_stages > 1
        self.is_data_parallel = self.grid.data_parallel_size > 1
        self.device = next((p.device for p in model.parameters()), None)
        if self.device is None:
            self.device = torch.device('cuda', torch.cuda.current_device()) if torch.cuda.is_available() else torch.device('cpu')
        self._micro_batch_size = int(self.config.get('train_micro_batch_size_per_gpu', 1))
        self.micro_batches = int(self.config.get('gradient_accumulation_steps', 1))
        self._gradient_clipping = float(self.config.get('gradient_clipping', 0.0))
        self.steps_per_print = int(self.config.get('steps_per_print', 10))
        self.optimizer = None
        self.lr_scheduler = None
        self.communication_data_type = None
        self.first_last_stage_group = None
        self._support_torch_style_backward = True
        self.global_steps = 0
        self.global_samples = 0
        self._grad_norm = None
        self.loss_fn = model.loss_fn
        self.pipe_buffers = {'inputs': [], 'labels': [], 'outputs': [], 'grads': []}
        # 'pipeline_schedule': '1f1b' (the reference's instruction stream) or 'zb' (split-backward zero-bubble order)
        self.pipeline_schedule = str(self.config.get('pipeline_schedule', '1f1b')).lower()
        self.zb_costs = tuple(self.config.get('zb_costs', (13, 17, 10)))
        self.zb_max_inflight = self.config.get('zb_max_inflight', None)
        # relative work per stage for the zero-bubble planner; default: the number of layers each stage holds, not counting
        # the model's first (embedding) and last (output head) layer, which are cheap next to a transformer block in every
        # model definition of the reference (models/flux.py:396-404, qwen_image.py:490-496, wan/wan.py:399-411)
        self.zb_stage_weights = self.config.get('zb_stage_weights', None)
        if self.zb_stage_weights is None and getattr(model, 'parts', None) is not None and len(model.parts) == self.num_stages + 1:
            n_layers = int(model.parts[-1])
            w = [int(model.parts[i + 1] - model.parts[i]) for i in range(self.num_stages)]
            if n_layers >= self.num_stages + 2:
                w[0] -= 1
                w[-1] -= 1
            self.zb_stage_weights = [max(1, x) for x in w]
        self._wgrad_queues = {}
        self._comm_stream = None                      # side stream of the data-parallel gradient all-reduce
        self._dp_reduced_layers, self._dp_reduced_ptrs = set(), set()
        self.dp_reduce_events = None
        self.dp_early_layers = 0                      # layers whose all-reduce started under the backward pass (last step)
        self.dp_overlap = bool(self.config.get('dp_overlap', os.environ.get('DPIPE_DP_OVERLAP', '1') != '0'))
        self._broadcast_model()
        self.link = self._make_link()
        self.total_loss = None
        self.fwd_losses = []
        self._data_iter = None
        self._busy_ms = 0.0

    def _broadcast_model(self):
        """utils/patches.py:163-172 (installed over DeepSpeedEngine._broadcast_model): at engine construction every
        data-parallel replica takes the TRAINABLE parameters of the first replica of its stage (frozen ones are loaded
        identically from disk and are not sent).  Parameters that alias one fused allocation are sent once."""
        if not self.is_data_parallel:
            return
        group = self.grid.get_data_parallel_group()
        src = self.grid.dp_group[0]
        seen = set()
        for p in self.module.parameters():
            if not p.requires_grad or p.data_ptr() in seen:
                continue
            seen.add(p.data_ptr())
            with torch.no_grad():
                # in place on the parameter itself (not `.data`): the version counter moves, so caches keyed on it
                # (lora.py: the fused [[W|B],[A|0]] site buffers) are rebuilt from the broadcast values
                dist.broadcast(p, src, group=group)
                p.add_(0)

    # ------------------------------------------------------------------ DeepSpeed-compatible accessors
    def is_first_stage(self):
        return self.stage_id == 0

    def is_last_stage(self):
        return self.stage_id == self.num_stages - 1

    def train_micro_batch_size_per_gpu(self):
        return self._micro_batch_size

    def gradient_accumulation_steps(self):
        return self.micro_batches

    def gradient_clipping(self):
        return self._gradient_clipping

    def train_batch_size(self):
        return self._micro_batch_size * self.micro_batches * self.grid.data_parallel_size

    def reset_activation_shape(self):
        """train.py:916 — boundary shapes may change between steps (resolution buckets)."""
        self.link.reset()

    def _configure_optimizer(self, client_optimizer, model_parameters):
        """train.py:817 — `client_optimizer` is a factory taking the trainable parameter list."""
        self.optimizer = client_optimizer(model_parameters) if callable(client_optimizer) else client_optimizer
        return self.optimizer

    def _make_link(self):
        """'auto' picks the CUDA-IPC link when every rank of the job sits on one host and sees the same GPUs under the same
        ordinals (the reference's launch: one node, `deepspeed --num_gpus=N`, README.md:118); anything else — several nodes,
        one CUDA_VISIBLE_DEVICES per rank — falls back to torch.distributed p2p with a notice.  The decision is taken from
        one all-gather so that every rank takes the same one."""
        kind = self.config.get('stage_link', 'auto')
        devices = None
        if kind == 'auto':
            kind = 'ipc' if (self.device.type == 'cuda' and self.is_pipe_parallel
                             and os.environ.get('DPIPE_STAGE_LINK', 'ipc') == 'ipc') else 'dist'
        if kind == 'ipc' and self.is_pipe_parallel:
            import socket
            mine = (socket.gethostname(), os.environ.get('CUDA_VISIBLE_DEVICES'), self.device.index, torch.cuda.device_count())
            seen = [None] * dist.get_world_size()
            dist.all_gather_object(seen, mine)
            ok = (len({x[0] for x in seen}) == 1 and len({x[1] for x in seen}) == 1
                  and all(x[2] is not None and x[2] < x[3] for x in seen))
            if not ok:
                if self.global_rank == 0:
                    print('stage link: the ranks are not on one host with a common view of its GPUs; using torch.distributed '
                          'p2p on the stage boundaries instead of CUDA-IPC peer copies', flush=True)
                kind = 'dist'
            else:
                devices = [x[2] for x in seen]
        if kind == 'ipc' and self.is_pipe_parallel:
            from .ipc_link import IpcLink
            return IpcLink(self, devices)
        if self.pipeline_schedule == 'zb' and self.is_pipe_parallel and self.device.type == 'cuda':
            # the split-backward order lets a stage run ahead of its neighbour, which needs one-sided sends.  NCCL
            # point-to-point operations between two ranks run in issue order on both sides: "send activation k+1" on one
            # stage and "send gradient k" on the other wait for each other's receive forever (seen on 2 GPUs).
            if self.global_rank == 0:
                print("pipeline_schedule 'zb' needs the one-sided CUDA-IPC stage link; with torch.distributed p2p on the "
                      "stage boundaries the reference's 1F1B order is used instead", flush=True)
            self.pipeline_schedule = '1f1b'
        return DistLink(self)

    # ------------------------------------------------------------------ public API
    def train_batch(self, data_iter=None):
        self.module.train()
        self.total_loss = None
        self.fwd_losses = []
        self._data_iter = data_iter
        self.dp_early_layers = 0
        if self.pipeline_schedule == 'zb':
            sched = ZeroBubbleSchedule(self.micro_batches, self.num_stages, self.stage_id, self.zb_costs, self.zb_max_inflight,
                                       self.zb_stage_weights)
        else:
            sched = TrainSchedule(self.micro_batches, self.num_stages, self.stage_id)
        self._reserve_buffers(sched.num_pipe_buffers())
        self._exec_schedule(sched, train=True)
        self.global_steps += 1
        self.global_samples += self.train_batch_size()
        loss = self._aggregate_total_loss(self.micro_batches)
        if self.steps_per_print and self.global_steps % self.steps_per_print == 0 and self.global_rank == 0:
            lr = self.optimizer.param_groups[0]['lr'] if self.optimizer and self.optimizer.param_groups else float('nan')
            print(f'steps: {self.global_steps} loss: {float(loss):.4f} lr: {lr:.3e}', flush=True)
        return loss

    def eval_batch(self, data_iter, num_micro_batches=None, return_logits=False, compute_loss=True, reduce_output='avg'):
        self.module.eval()
        n = num_micro_batches or self.micro_batches
        self.total_loss = None
        self.fwd_losses = []
        self._data_iter = data_iter
        sched = InferenceSchedule(n, self.num_stages, self.stage_id)
        self._reserve_buffers(sched.num_pipe_buffers())
        with torch.no_grad():
            self._exec_schedule(sched, train=False)
        return self._aggregate_total_loss(n)

    # ------------------------------------------------------------------ schedule execution
    def _reserve_buffers(self, n):
        for k in self.pipe_buffers:
            if len(self.pipe_buffers[k]) < n:
                self.pipe_buffers[k].extend([None] * (n - len(self.pipe_buffers[k])))

    def _exec_schedule(self, sched, train):
        if getattr(self.link, 'native', False):
            return self._exec_schedule_native(sched, train)
        handlers = self._INSTRUCTION_MAP
        for tick in sched.steps():
            for cmd in tick:
                handlers[type(cmd)](self, cmd, train)
        self.link.flush()

    def _exec_schedule_native(self, sched, train):
        """The C++ executor (csrc/stage_exec.cu) walks the instruction stream: it runs every Send / Recv itself (copy stream,
        events, peer copies, device-side flags) and hands back only the instructions that need autograd or the optimizer,
        plus — once per step and channel — the host handshake of a receiving channel."""
        import ctypes
        from .. import _lib
        from .ipc_link import CH_ACT_IN, CH_GRAD_IN, OP_NEED_HANDSHAKE
        from .schedule import _Instr, make_instruction
        lib = _lib.lib()
        plan = sched.raw()
        ex = self.link.exec
        _lib.check(lib.dpipe_exec_load_plan(ex, plan, len(plan), int(train), int(self.is_first_stage()), int(self.is_last_stage()),
                                            max(1, len(self.pipe_buffers['inputs']))), 'dpipe_exec_load_plan')
        handlers = self._INSTRUCTION_MAP
        ins = _Instr()
        while True:
            stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
            rc = lib.dpipe_exec_next(ex, stream, ctypes.byref(ins))
            if rc == 0:
                break
            _lib.check(0 if rc > 0 else rc, 'dpipe_exec_next')
            if ins.op >= OP_NEED_HANDSHAKE:
                cid = ins.op - OP_NEED_HANDSHAKE
                if cid not in (CH_ACT_IN, CH_GRAD_IN):
                    raise RuntimeError('stage executor: a Send was reached before its tuple was staged (internal error)')
                like = None
                if cid == CH_GRAD_IN:
                    like = [t for t in self.pipe_buffers['outputs'][ins.buffer] if t.is_floating_point()]
                self.link.handshake_recv(cid, like)
                continue
            cmd = make_instruction(ins.op, ins.buffer, ins.micro_batch)
            handlers[type(cmd)](self, cmd, train)

    def _exec_load_micro_batch(self, cmd, train):
        b = cmd.buffer_id
        batch = next(self._data_iter)
        if self.is_first_stage():
            feats = batch[0]
            if torch.is_tensor(feats):
                feats = (feats,)
            loaded = []
            for x in feats:
                assert torch.is_tensor(x)
                # a private copy on the device, like the reference's `clone().detach().to(device)` — but a host tensor is
                # copied ONCE (pinned memory: asynchronously), never cloned into pageable memory first
                y = x.detach()
                y = y.clone() if y.device == self.device else y.to(self.device, non_blocking=True)
                y.requires_grad = y.is_floating_point() and train
                loaded.append(y)
            self.pipe_buffers['inputs'][b] = tuple(loaded)
        if self.is_last_stage():
            labels = batch[1]
            if torch.is_tensor(labels):
                labels = labels.to(self.device, non_blocking=True)
            else:
                labels = tuple(x.to(self.device, non_blocking=True) for x in labels)
            self.pipe_buffers['labels'][b] = labels

    def _exec_forward_pass(self, cmd, train):
        b = cmd.buffer_id
        inputs = self.pipe_buffers['inputs'][b]
        # 1F1B runs the backward passes in micro-batch order: the gradients a layer holds after the backward of the LAST
        # micro-batch are final, and the data-parallel all-reduce of that layer may start while earlier layers still compute
        arm = (train and self.is_data_parallel and self.dp_overlap and self.pipeline_schedule != 'zb'
               and getattr(cmd, 'micro_batch_id', -1) == self.micro_batches - 1)
        self.module._grads_ready_cb = self._dp_reduce_layers if arm else None
        try:
            outputs = self.module(inputs if len(inputs) > 1 else inputs[0])
        finally:
            self.module._grads_ready_cb = None
        if self.is_last_stage():
            if self.loss_fn is not None:
                loss = self.loss_fn(outputs, self.pipe_buffers['labels'][b])
            else:
                loss = outputs
            self.pipe_buffers['outputs'][b] = loss
            self.fwd_losses.append(loss.detach())
            self.total_loss = loss.detach().clone() if self.total_loss is None else self.total_loss + loss.detach()
        else:
            if torch.is_tensor(outputs):
                outputs = (outputs,)
            self.pipe_buffers['outputs'][b] = tuple(outputs)
            if getattr(self.link, 'native', False):
                from .ipc_link import CH_ACT_OUT
                self.link.stage(CH_ACT_OUT, b, self.pipe_buffers['outputs'][b])
                if not train:
                    self.pipe_buffers['outputs'][b] = None       # (the link keeps the tuple alive until it has been copied)
        if not train:
            self.pipe_buffers['inputs'][b] = None
            if self.is_last_stage():
                # forward-only: the loss is already in total_loss, nothing will come back for this buffer
                self.pipe_buffers['outputs'][b] = None
                self.pipe_buffers['labels'][b] = None
                if not self.is_first_stage() and not getattr(self.link, 'native', False):
                    self.link.release_activations(b, cmd.micro_batch_id)

    def _exec_backward_input(self, cmd, train):
        """split backward: weight-gradient work of the layers that support it is queued instead of launched.
        Contract for the queued closures (ops.defer): they may capture tensors the block produced, never tensors RECEIVED
        from another stage — a received tensor is a view of a stage-link mailbox slot that is released to the sender as
        soon as this pass (and its SendGrad) is enqueued.  wan.py clones the one boundary tensor it needs (`context`)."""
        from .. import ops
        q = []
        ops.WGRAD_DEFER = q
        try:
            self._exec_backward_pass(cmd, train)
        finally:
            ops.WGRAD_DEFER = None
        self._wgrad_queues[cmd.micro_batch_id] = q

    def _exec_backward_weight(self, cmd, train):
        with torch.no_grad():          # the queued closures are the tail of a backward pass: never recorded by autograd
            for fn in self._wgrad_queues.pop(cmd.micro_batch_id, ()):
                fn()

    def _exec_backward_pass(self, cmd, train):
        b = cmd.buffer_id
        outputs = self.pipe_buffers['outputs'][b]
        if self.is_last_stage():
            (outputs / self.micro_batches).backward()
        else:
            grads = self.pipe_buffers['grads'][b]
            outs = [t for t in outputs if t.is_floating_point()]
            assert len(outs) == len(grads)
            pairs = [(t, g) for t, g in zip(outs, grads) if t.requires_grad]
            torch.autograd.backward(tensors=[p[0] for p in pairs], grad_tensors=[p[1] for p in pairs])
            if not getattr(self.link, 'native', False):
                self.link.release_grads(b, cmd.micro_batch_id)     # (the C++ executor hands the slot back itself)
        self.pipe_buffers['outputs'][b] = None
        self.pipe_buffers['grads'][b] = None
        self.pipe_buffers['labels'][b] = None
        if getattr(self.link, 'native', False) and not self.is_first_stage():
            from .ipc_link import CH_GRAD_OUT
            self.link.stage(CH_GRAD_OUT, b, self._input_grads(b))   # for the SendGrad the executor runs next
            self.pipe_buffers['inputs'][b] = None

    def _exec_send_activations(self, cmd, train):
        b = cmd.buffer_id
        self.link.send_activations(self.pipe_buffers['outputs'][b], b, cmd.micro_batch_id, keep=train)
        if not train:
            self.pipe_buffers['outputs'][b] = None

    def _exec_recv_activations(self, cmd, train):
        b = cmd.buffer_id
        if getattr(self.link, 'native', False):
            from .ipc_link import CH_ACT_IN
            tensors = self.link.wrap(CH_ACT_IN, cmd.micro_batch_id)   # the executor has already made the stream wait for it
        else:
            tensors = self.link.recv_activations(b, cmd.micro_batch_id)
        out = []
        for t in tensors:
            t = t.detach()
            t.requires_grad = t.is_floating_point() and train
            out.append(t)
        self.pipe_buffers['inputs'][b] = tuple(out)

    def _input_grads(self, b):
        """gradients of every floating-point tensor of the stage's input tuple (zeros where autograd produced none: the
        previous stage expects one gradient per float output, SURVEY 8a E6)"""
        grads = []
        for t in self.pipe_buffers['inputs'][b]:
            if t.is_floating_point():
                grads.append(t.grad if t.grad is not None else torch.zeros_like(t))
        return tuple(grads)

    def _exec_send_grads(self, cmd, train):
        b = cmd.buffer_id
        self.link.send_grads(self._input_grads(b), b, cmd.micro_batch_id)
        self.pipe_buffers['inputs'][b] = None

    def _exec_recv_grads(self, cmd, train):
        b = cmd.buffer_id
        outputs = self.pipe_buffers['outputs'][b]
        like = [t for t in outputs if t.is_floating_point()]
        if getattr(self.link, 'native', False):
            from .ipc_link import CH_GRAD_IN
            self.pipe_buffers['grads'][b] = self.link.wrap(CH_GRAD_IN, cmd.micro_batch_id)
        else:
            self.pipe_buffers['grads'][b] = self.link.recv_grads(like, b, cmd.micro_batch_id)

    def _exec_reduce_tied_grads(self, cmd, train):
        pass   # no tied layers in any reference model definition

    # ------------------------------------------------------------------ data-parallel gradient all-reduce (E7)
    def _dp_reduce_buffers(self, grads):
        """mean over the data-parallel group of every tensor in `grads`, in place.  Large contiguous buffers (the fused
        weight-gradient allocations) go one collective each; small ones are coalesced.  NCCL averages inside the collective
        (ReduceOp.AVG); other backends sum and divide."""
        group = self.grid.get_data_parallel_group()
        world = self.grid.data_parallel_size
        comm_dtype = self.communication_data_type
        avg = bool(grads) and grads[0].is_cuda and 'nccl' in str(dist.tdist.get_backend(group))
        op = dist.ReduceOp.AVG if avg else dist.ReduceOp.SUM
        small, small_elems = [], 0

        def flush_small():
            nonlocal small, small_elems
            if not small:
                return
            flat = torch.cat([g.reshape(-1).to(comm_dtype or g.dtype) for g in small])
            dist.all_reduce(flat, op=op, group=group)
            if not avg:
                flat.div_(world)
            off = 0
            for g in small:
                g.copy_(flat[off:off + g.numel()].view_as(g))
                off += g.numel()
            small, small_elems = [], 0

        for g in grads:
            if g.numel() >= (1 << 20) and g.is_contiguous() and (comm_dtype is None or comm_dtype == g.dtype):
                dist.all_reduce(g, op=op, group=group)
                if not avg:
                    g.div_(world)
            else:
                small.append(g)
                small_elems += g.numel()
                if small_elems >= (1 << 24):
                    flush_small()
        flush_small()

    def _dp_reduce_layers(self, first, last, early=True):
        """all-reduce the gradients of local layers [first, last) that have not been reduced in this step.  On CUDA the
        collectives are enqueued on a side stream ordered after everything the compute stream holds right now, so they
        run under the backward passes of the layers still to come (utils/patches.py:152-156 reduces after the drain)."""
        params = []
        for i in range(first, last):
            if early:
                if i in self._dp_reduced_layers:
                    continue
                self._dp_reduced_layers.add(i)
                self.dp_early_layers += 1
            # (the final pass looks at every layer again: a gradient that did not exist yet when the layer's callback ran is
            # picked up here; what has been reduced is remembered per buffer, not per layer)
            f = self.module.forward_funcs[i]
            if isinstance(f, torch.nn.Module):
                params += [p for p in f.parameters() if p.requires_grad and p.grad is not None]
        grads = [g for g in self._unique_grad_buffers(params) if g.data_ptr() not in self._dp_reduced_ptrs]
        if not grads:
            return
        self._dp_reduced_ptrs.update(g.data_ptr() for g in grads)
        if self.device.type != 'cuda':
            self._dp_reduce_buffers(grads)
            return
        if self._comm_stream is None:
            self._comm_stream = torch.cuda.Stream(device=self.device)
        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream())
        with torch.cuda.stream(self._comm_stream):
            self._comm_stream.wait_event(ev)
            self._dp_reduce_buffers(grads)

    def _exec_reduce_grads(self, cmd, train):
        if not self.is_data_parallel:
            return
        cuda = self.device.type == 'cuda'
        if cuda:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        self._dp_reduce_layers(0, len(self.module.forward_funcs), early=False)      # whatever the backward hooks did not start
        if cuda and self._comm_stream is not None:
            done = torch.cuda.Event()
            done.record(self._comm_stream)
            torch.cuda.current_stream().wait_event(done)
            e1.record()
            self.dp_reduce_events = (e0, e1)     # elapsed = the part of the all-reduce the step actually waited for
        self._dp_reduced_layers.clear()
        self._dp_reduced_ptrs.clear()

    @staticmethod
    def _unique_grad_buffers(params):
        """the gradient storage behind `params`, every byte once: per-projection views of one fused buffer collapse into
        that buffer (flux_blocks.FusedParam), everything else is the .grad tensor itself"""
        out, seen = [], set()
        for p in params:
            g = p.grad
            if g is None:
                continue
            base = g._base if g._base is not None else g
            if base is not g and base.is_contiguous() and base.dtype == g.dtype:
                g = base
            key = (g.data_ptr(), g.numel())
            if key in seen:
                continue
            seen.add(key)
            out.append(g.detach())
        return out

    def _clip_grad_norm(self, params, max_norm):
        """utils/patches.py:175-246: sqrt(sum of squared per-parameter fp32 norms) over the whole pipeline, then
        g *= min(1, max_norm / (norm + 1e-6)).  On the device both passes are one multi-tensor kernel each
        (csrc/step_tail.cu): no fp32 copies of the gradients, and no pass at all over them when nothing is clipped."""
        from .. import ops
        grads = PipelineEngine._unique_grad_buffers(params)
        fused = bool(grads) and ops.grads_supported(grads) and PipelineEngine._fused_views_cover(params, grads)
        if not fused:
            grads = [p.grad for p in params if p.grad is not None]
        if fused:
            total = ops.grad_sumsq(grads)
        elif grads:
            norms = torch._foreach_norm([g.detach().float() if g.dtype != torch.float32 else g.detach() for g in grads])
            total = torch.stack(norms).square().sum().float()
        else:
            total = torch.zeros((), dtype=torch.float32, device=self.device)
        total = total.to(self.device)
        if self.is_pipe_parallel:
            dist.all_reduce(total, op=dist.ReduceOp.SUM, group=self.grid.get_pipe_parallel_group())
        total_norm = total.sqrt()
        if self.is_data_parallel:
            # the reference averages the (identical) norm over the data-parallel group
            scaled = total_norm / float(self.grid.data_parallel_size)
            dist.all_reduce(scaled, group=self.grid.get_data_parallel_group())
            total_norm = scaled
        clip_coef = torch.clamp(max_norm / (total_norm + 1e-6), max=1.0)
        if fused:
            ops.grad_scale(grads, clip_coef.float().reshape(1).contiguous())
        elif grads:
            torch._foreach_mul_(grads, clip_coef.to(grads[0].device))
        return total_norm

    @staticmethod
    def _fused_views_cover(params, buffers):
        """a fused buffer may be summed as a whole only if its views cover it (they do: FusedParam slices the whole
        allocation; checked by element count so that a partially trainable fused weight falls back to the per-tensor path)"""
        return sum(b.numel() for b in buffers) == sum(p.grad.numel() for p in params if p.grad is not None)

    def _exec_optimizer_step(self, cmd, train):
        params = [p for p in self.module.parameters() if p.requires_grad]
        if self._gradient_clipping > 0.0:
            self._grad_norm = self._clip_grad_norm(params, self._gradient_clipping)
            if self.optimizer is not None:
                self.optimizer._grad_norm = self._grad_norm
        if self.optimizer is not None:
            self.optimizer.step()
            self.optimizer.zero_grad(set_to_none=True)
        else:
            for p in params:
                p.grad = None
        if self.lr_scheduler is not None:
            self.lr_scheduler.step()

    _INSTRUCTION_MAP = {
        OptimizerStep: _exec_optimizer_step,
        ReduceGrads: _exec_reduce_grads,
        ReduceTiedGrads: _exec_reduce_tied_grads,
        LoadMicroBatch: _exec_load_micro_batch,
        ForwardPass: _exec_forward_pass,
        BackwardPass: _exec_backward_pass,
        BackwardInput: _exec_backward_input,
        BackwardWeight: _exec_backward_weight,
        SendActivation: _exec_send_activations,
        RecvActivation: _exec_recv_activations,
        SendGrad: _exec_send_grads,
        RecvGrad: _exec_recv_grads,
    }

    # ------------------------------------------------------------------ loss aggregation (E10)
    def _aggregate_total_loss(self, num_micro_batches):
        if self.is_last_stage():
            loss = (self.total_loss / num_micro_batches).float().reshape(1).to(self.device)
            if self.is_data_parallel:
                dist.all_reduce(loss, group=self.grid.get_data_parallel_group())
                loss /= self.grid.data_parallel_size
        else:
            loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        if self.is_pipe_parallel:
            src = self.grid.stage_to_global(self.num_stages - 1)
            dist.broadcast(loss, src, group=self.grid.get_pipe_parallel_group())
        return loss.reshape(())

    # ------------------------------------------------------------------ checkpoint (SURVEY 8f.1)
    def save_checkpoint(self, save_dir, tag=None, client_state=None, save_latest=True, exclude_frozen_parameters=False):
        tag = tag or f'global_step{self.global_steps}'
        path = os.path.join(save_dir, tag)
        os.makedirs(path, exist_ok=True)
        sd = {}
        for name, p in self.module.named_parameters():
            if exclude_frozen_parameters and not p.requires_grad:
                continue
            sd[getattr(p, 'original_name', name)] = p.detach().cpu()
        state = {
            'module': sd,
            'optimizer': self.optimizer.state_dict() if self.optimizer is not None else None,
            'lr_scheduler': self.lr_scheduler.state_dict() if self.lr_scheduler is not None else None,
            'global_steps': self.global_steps,
            'global_samples': self.global_samples,
            'client_state': client_state or {},
        }
        fn = os.path.join(path, f'stage_{self.stage_id:02d}-dp_{self.grid.data_parallel_id:02d}_states.pt')
        if self.grid.data_parallel_id == 0 or self.optimizer is not None:
            torch.save(state, fn)
        dist.barrier()
        if save_latest and self.global_rank == 0:
            with open(os.path.join(save_dir, 'latest'), 'w') as f:
                f.write(tag)
        return True

    def load_checkpoint(self, load_dir, tag=None, load_module_strict=True, load_optimizer_states=True,
                        load_lr_scheduler_states=True):
        if tag is None:
            latest = os.path.join(load_dir, 'latest')
            if not os.path.isfile(latest):
                return None, None
            with open(latest) as f:
                tag = f.read().strip()
        fn = os.path.join(load_dir, tag, f'stage_{self.stage_id:02d}-dp_{self.grid.data_parallel_id:02d}_states.pt')
        if not os.path.isfile(fn):
            fn = os.path.join(load_dir, tag, f'stage_{self.stage_id:02d}-dp_00_states.pt')
        state = torch.load(fn, map_location='cpu', weights_only=False)
        by_name = {getattr(p, 'original_name', n): p for n, p in self.module.named_parameters()}
        missing = []
        for k, p in by_name.items():
            if k in state['module']:
                with torch.no_grad():
                    p.copy_(state['module'][k])      # in place on the parameter itself: bumps its version counter (lora.py watches it)
            elif p.requires_grad:
                missing.append(k)
        if load_module_strict and missing:
            raise RuntimeError(f'checkpoint is missing parameters: {missing[:5]}')
        if load_optimizer_states and self.optimizer is not None and state.get('optimizer') is not None:
            self.optimizer.load_state_dict(state['optimizer'])
        if load_lr_scheduler_states and self.lr_scheduler is not None and state.get('lr_scheduler') is not None:
            self.lr_scheduler.load_state_dict(state['lr_scheduler'])
        self.global_steps = state.get('global_steps', 0)
        self.global_samples = state.get('global_samples', 0)
        return os.path.join(load_dir, tag), state.get('client_state', {})


def initialize(args=None, model=None, config=None, **kwargs):
    """deepspeed.initialize(args=, model=, config=) -> (engine, optimizer, None, None)   (train.py:623-627)."""
    engine = PipelineEngine(model, config, args=args)
    return engine, engine.optimizer, None, None
