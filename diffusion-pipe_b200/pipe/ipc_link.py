"""IpcLink — the single-node stage-boundary transport: CUDA-IPC mailboxes + cudaMemcpyPeerAsync over NVLink + device-side
sequence flags.  No NCCL on the boundary.  The data path lives in C++ (csrc/stage_exec.cu: dpipe_exec_*): the executor
walks the stage's instruction stream and runs every Send / Recv itself on its own copy stream and events; this module is
the HOST control plane only — mailbox allocation, the once-per-step shape / IPC-handle handshake over a gloo side group,
and wrapping a received slot into tensors.

Per direction (activations stage s -> s+1, gradients s+1 -> s) there is one channel:
  * the RECEIVER owns a mailbox  [ready flags | NSLOTS x slot]  in its own HBM and exports it once (re-exported only
    if a larger boundary tuple shows up: resolution buckets change shapes between steps, train.py:916);
  * the SENDER owns the matching `free` flag array.
  send  (sender's copy stream):   wait free[k] >= w-1 ; peer-copy every tensor into slot k ; ready[k] = w
  recv  (receiver's compute stream): wait ready[k] >= w ; the tensors ARE views of slot k (no second copy)
  release (receiver's compute stream, once the slot's consumer has run): free[k] = w
with k = micro_batch % NSLOTS and w the per-slot use count.  The host never blocks on the data path; it only exchanges
shapes / IPC handles over a gloo side group the first time after `reset_activation_shape()` (once per step, like the
reference's metadata handshake) — host metadata, no device synchronisation.

Replaces DeepSpeed's p2p send/recv of the boundary tuple (SURVEY.md 8a E6, schedule at utils/patches.py:134-143).
"""
import ctypes
import os

import torch
import torch.distributed as tdist

from .. import _lib

_DTYPES = [torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.int32, torch.int16, torch.int8, torch.uint8,
           torch.bool, torch.float64]
_DTYPE_ID = {d: i for i, d in enumerate(_DTYPES)}
_META_LEN = 192
_ALIGN = 256
_WAIT_TIMEOUT_S = float(os.environ.get('DPIPE_LINK_TIMEOUT_S', 300.0))   # device-side flag wait; 0 = wait forever


def _align(n):
    return (n + _ALIGN - 1) // _ALIGN * _ALIGN


class _DevMem:
    """exposes a raw device allocation to torch through __cuda_array_interface__"""

    def __init__(self, ptr, nbytes):
        self.__cuda_array_interface__ = {'shape': (nbytes,), 'typestr': '|u1', 'data': (ptr, False), 'version': 2}


def _lib_call(name, *args):
    _lib.check(getattr(_lib.lib(), name)(*args), name)


def _ipc_alloc(nbytes):
    ptr = ctypes.c_void_p()
    handle = (ctypes.c_ubyte * 64)()
    _lib_call('dpipe_ipc_alloc', nbytes, ctypes.byref(ptr), handle)
    return ptr.value, bytes(handle)


def _ipc_open(handle):
    ptr = ctypes.c_void_p()
    buf = (ctypes.c_ubyte * 64).from_buffer_copy(handle)
    _lib_call('dpipe_ipc_open', buf, ctypes.byref(ptr))
    return ptr.value


def _layout(specs):
    """byte offset of every tensor inside a slot and the slot size"""
    offs, off = [], 0
    for dt, shape in specs:
        n = 1
        for s in shape:
            n *= s
        offs.append(off)
        off += _align(max(1, n * torch.empty((), dtype=dt).element_size()))
    return offs, off


class _Channel:
    def __init__(self, link, peer_rank, peer_device, sending, tag, cid):
        self.link = link
        self.cid = cid             # DPIPE_CH_* of include/dpipe.h
        self.remade = True         # the mailbox behind this channel is new: the executor restarts its slot counters
        self.peer_rank, self.peer_device = peer_rank, peer_device
        self.sending = sending
        self.tag = tag
        self.nslots = link.nslots
        self.flag_bytes = _align(8 * self.nslots)
        self.slot_bytes = 0
        self.specs = None          # [(dtype, shape)] valid until the next reset
        self.offs = None
        self.handshaken = False
        if sending:
            self.free_ptr, self.free_handle = _ipc_alloc(self.flag_bytes)    # flow-control flags live with the sender
            self.remote_ptr = None                                            # receiver's mailbox, mapped
        else:
            self.mail_ptr = None                                              # own mailbox
            self.mail_handle = None
            self.mail_u8 = None
            self.remote_free = None                                           # sender's free flags, mapped

    # ---- host-side control plane (gloo) ----
    def _send_cpu(self, t, tag):
        tdist.send(t, self.peer_rank, group=self.link.ctrl_group, tag=self.tag + tag)

    def _recv_cpu(self, t, tag):
        tdist.recv(t, self.peer_rank, group=self.link.ctrl_group, tag=self.tag + tag)

    def _ensure_mailbox(self, slot_bytes):
        """receiver: (re)allocate the mailbox if the boundary tuple outgrew it; returns True if it changed"""
        if self.mail_ptr is not None and slot_bytes <= self.slot_bytes:
            return False
        if self.mail_ptr is not None:
            torch.cuda.synchronize()
            _lib_call('dpipe_ipc_free', ctypes.c_void_p(self.mail_ptr))
            self.remade = True
        self.slot_bytes = _align(int(slot_bytes * 1.0))
        total = self.flag_bytes + self.nslots * self.slot_bytes
        self.mail_ptr, self.mail_handle = _ipc_alloc(total)
        self.mail_u8 = torch.as_tensor(_DevMem(self.mail_ptr, total), device=self.link.device)
        return True

    def _map_mailbox(self, handle, slot_bytes):
        if self.remote_ptr is not None:
            torch.cuda.synchronize()
            _lib_call('dpipe_ipc_close', ctypes.c_void_p(self.remote_ptr))
            self.remade = True
            # the receiver starts the new mailbox with zeroed flags: restart our own flow-control flags as well
            self.link._zero(self.free_ptr, self.flag_bytes)
        self.remote_ptr = _ipc_open(handle)
        self.slot_bytes = slot_bytes

    # ---- activations: the sender describes the tuple ----
    def handshake_send_described(self, tensors):
        meta = torch.zeros(_META_LEN, dtype=torch.int64)
        vals = [len(tensors), 0 if self.handshaken else 1]
        for t in tensors:
            vals += [_DTYPE_ID[t.dtype], t.dim()] + list(t.shape)
        assert len(vals) <= _META_LEN, 'boundary tuple too complex for the metadata message'
        meta[:len(vals)] = torch.tensor(vals, dtype=torch.int64)
        self._send_cpu(meta, 0)
        if not self.handshaken:
            self._send_cpu(torch.frombuffer(bytearray(self.free_handle), dtype=torch.uint8), 1)
        reply = torch.zeros(4, dtype=torch.int64)
        self._recv_cpu(reply, 2)
        if int(reply[0]):
            h = torch.zeros(64, dtype=torch.uint8)
            self._recv_cpu(h, 3)
            self._map_mailbox(bytes(h.numpy().tobytes()), int(reply[1]))
        self.handshaken = True
        self.specs = [(t.dtype, tuple(t.shape)) for t in tensors]
        self.offs, _ = _layout(self.specs)
        self.bind(self.remade)
        self.remade = False

    def handshake_recv_described(self):
        meta = torch.zeros(_META_LEN, dtype=torch.int64)
        self._recv_cpu(meta, 0)
        m = meta.tolist()
        n, first = m[0], m[1]
        if first:
            h = torch.zeros(64, dtype=torch.uint8)
            self._recv_cpu(h, 1)
            self.remote_free = _ipc_open(bytes(h.numpy().tobytes()))
        specs, pos = [], 2
        for _ in range(n):
            dt, nd = _DTYPES[m[pos]], m[pos + 1]
            specs.append((dt, tuple(m[pos + 2:pos + 2 + nd])))
            pos += 2 + nd
        self.specs = specs
        self.offs, need = _layout(specs)
        changed = self._ensure_mailbox(need)
        self._send_cpu(torch.tensor([1 if changed else 0, self.slot_bytes, self.nslots, 0], dtype=torch.int64), 2)
        if changed:
            self._send_cpu(torch.frombuffer(bytearray(self.mail_handle), dtype=torch.uint8), 3)
        self.handshaken = True
        self.bind(self.remade)
        self.remade = False

    # ---- gradients: the receiver already knows the shapes (its own outputs) ----
    def handshake_recv_known(self, like):
        self.specs = [(t.dtype, tuple(t.shape)) for t in like]
        self.offs, need = _layout(self.specs)
        changed = self._ensure_mailbox(need)
        self._send_cpu(torch.tensor([1 if changed else 0, self.slot_bytes, self.nslots, 0 if self.handshaken else 1],
                                    dtype=torch.int64), 0)
        if changed:
            self._send_cpu(torch.frombuffer(bytearray(self.mail_handle), dtype=torch.uint8), 1)
        if not self.handshaken:
            h = torch.zeros(64, dtype=torch.uint8)
            self._recv_cpu(h, 2)
            self.remote_free = _ipc_open(bytes(h.numpy().tobytes()))
        self.handshaken = True
        self.bind(self.remade)
        self.remade = False

    def handshake_send_known(self, tensors):
        info = torch.zeros(4, dtype=torch.int64)
        self._recv_cpu(info, 0)
        if int(info[0]):
            h = torch.zeros(64, dtype=torch.uint8)
            self._recv_cpu(h, 1)
            self._map_mailbox(bytes(h.numpy().tobytes()), int(info[1]))
        if int(info[3]):
            self._send_cpu(torch.frombuffer(bytearray(self.free_handle), dtype=torch.uint8), 2)
        self.handshaken = True
        self.specs = [(t.dtype, tuple(t.shape)) for t in tensors]
        self.offs, _ = _layout(self.specs)
        self.bind(self.remade)
        self.remade = False

    # ---- after a handshake: hand the channel to the C++ executor ----
    def bind(self, reset_counts):
        ex = self.link.exec
        if self.sending:
            _lib_call('dpipe_exec_bind', ex, self.cid, ctypes.c_void_p(self.free_ptr), ctypes.c_void_p(self.remote_ptr),
                      self.peer_device, self.flag_bytes, self.slot_bytes, int(reset_counts))
        else:
            _lib_call('dpipe_exec_bind', ex, self.cid, ctypes.c_void_p(self.mail_ptr), ctypes.c_void_p(self.remote_free),
                      self.peer_device, self.flag_bytes, self.slot_bytes, int(reset_counts))
        n = len(self.specs)
        sizes = []
        for dt, shape in self.specs:
            k = 1
            for x in shape:
                k *= x
            sizes.append(k * torch.empty((), dtype=dt).element_size())
        self.nbytes = sizes
        _lib_call('dpipe_exec_set_layout', ex, self.cid, n, (ctypes.c_int64 * n)(*self.offs), (ctypes.c_int64 * n)(*sizes))

    def wrap(self, mb):
        """the tensors of the tuple received for micro-batch mb: views of the mailbox slot (no second copy)"""
        base = ctypes.c_void_p()
        _lib_call('dpipe_exec_recv_base', self.link.exec, self.cid, mb, ctypes.byref(base))
        off0 = base.value - self.mail_ptr
        out = []
        for (dt, shape), off, nbytes in zip(self.specs, self.offs, self.nbytes):
            out.append(self.mail_u8[off0 + off: off0 + off + nbytes].view(dt).view(shape))
        return out


CH_ACT_OUT, CH_ACT_IN, CH_GRAD_OUT, CH_GRAD_IN = 0, 1, 2, 3        # include/dpipe.h DPIPE_CH_*
OP_NEED_HANDSHAKE = 100


class IpcLink:
    native = True      # the engine runs its schedule through dpipe_exec_next (pipe/engine.py:_exec_schedule_native)

    def __init__(self, engine, rank_devices=None):
        """rank_devices[r] = CUDA ordinal of global rank r (engine._make_link gathers them); None = ordinal follows the rank"""
        self.engine = engine
        self.device = engine.device
        assert self.device.type == 'cuda'
        grid = engine.grid
        # 1F1B keeps at most `stages` micro-batches in flight on a stage; the zero-bubble order holds up to
        # `zb_max_inflight` (default 2 x stages).  A receiver that may hold n un-released activations needs n slots:
        # with fewer, the sender would wait for a slot whose release is ordered AFTER the forward pass it is feeding.
        self.nslots = max(2, engine.num_stages)
        if engine.pipeline_schedule == 'zb':
            self.nslots = max(2 * self.nslots, int(engine.zb_max_inflight or 2 * engine.num_stages))
        self.exec = ctypes.c_void_p()
        _lib_call('dpipe_exec_create', self.device.index, self.nslots, _WAIT_TIMEOUT_S, ctypes.byref(self.exec))
        # the executor's copy stream, known to torch's allocator (record_stream on the tensors a pending copy still reads)
        self.copy_stream = torch.cuda.ExternalStream(_lib.lib().dpipe_exec_copy_stream(self.exec), device=self.device)
        # host control plane: one gloo group per pipeline (every rank creates all of them, in the same order)
        self.ctrl_group = None
        for d in range(grid.data_parallel_size):
            ranks = [grid._topo.get_rank(s, d) for s in range(grid.pipe_parallel_size)]
            g = tdist.new_group(ranks=ranks, backend='gloo')
            if d == grid.data_parallel_id:
                self.ctrl_group = g
        # peers: same node, all GPUs visible in every process under the same ordinals (two stages may share one device:
        # the peer copy degenerates to a device-local copy — tests/test_stage_link_one_gpu.py)
        local_rank = self.device.index

        def peer(stage):
            r = grid.stage_to_global(stage)
            return r, (rank_devices[r] if rank_devices is not None else local_rank + (r - engine.global_rank))
        s = engine.stage_id
        last = engine.num_stages - 1
        self.channels = {
            CH_ACT_OUT: _Channel(self, *peer(s + 1), sending=True, tag=100, cid=CH_ACT_OUT) if s < last else None,
            CH_ACT_IN: _Channel(self, *peer(s - 1), sending=False, tag=100, cid=CH_ACT_IN) if s > 0 else None,
            CH_GRAD_OUT: _Channel(self, *peer(s - 1), sending=True, tag=200, cid=CH_GRAD_OUT) if s > 0 else None,
            CH_GRAD_IN: _Channel(self, *peer(s + 1), sending=False, tag=200, cid=CH_GRAD_IN) if s < last else None,
        }
        self._fresh = {}
        self._keep = {}            # (channel, pipe buffer) -> the tensors a pending send still reads
        self.reset()

    def close(self):
        """explicit teardown (after a device synchronisation).  Not done from __del__: at interpreter exit torch's caching
        allocator may still hold events recorded on the executor's copy stream, and destroying the stream under it turns a
        clean exit into a CUDA error."""
        if self.exec:
            torch.cuda.synchronize()
            _lib.lib().dpipe_exec_destroy(self.exec)
            self.exec = ctypes.c_void_p()

    def _zero(self, ptr, nbytes):
        torch.as_tensor(_DevMem(ptr, nbytes), device=self.device).zero_()
        torch.cuda.synchronize()

    def reset(self):
        """engine.reset_activation_shape() (train.py:916): the next step re-announces its boundary tuples"""
        self._fresh = {c: True for c in self.channels}
        _lib_call('dpipe_exec_forget_layouts', self.exec)

    # ---- what the engine calls around the executor ----
    def stage(self, cid, buf, tensors):
        """the tuple a coming SendActivation / SendGrad of pipe buffer `buf` will copy; the first one of a step announces
        shapes (and, when a mailbox is new, IPC handles) to the neighbour over the gloo side group"""
        ch = self.channels[cid]
        ts = [t.contiguous() for t in tensors]
        if self._fresh[cid]:
            (ch.handshake_send_described if cid == CH_ACT_OUT else ch.handshake_send_known)(ts)
            self._fresh[cid] = False
        elif ch.specs != [(t.dtype, tuple(t.shape)) for t in ts]:
            # the slot layout on both sides comes from the handshake: a different tuple would be copied to wrong offsets
            raise RuntimeError('the boundary tuple changed shape or dtype since it was announced to the next stage: call '
                               'engine.reset_activation_shape() before a step whose micro-batches have new shapes '
                               '(train.py:916, train.py:181)')
        n = len(ts)
        _lib_call('dpipe_exec_stage_send', self.exec, cid, buf, n, (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts]))
        for t in ts:
            if t.numel():
                t.record_stream(self.copy_stream)
        self._keep[(cid, buf)] = ts

    def handshake_recv(self, cid, like=None):
        """DPIPE_OP_NEED_HANDSHAKE for a receiving channel (first Recv of a step)"""
        ch = self.channels[cid]
        if cid == CH_ACT_IN:
            ch.handshake_recv_described()
        else:
            ch.handshake_recv_known(like)
        self._fresh[cid] = False

    def wrap(self, cid, mb):
        return self.channels[cid].wrap(mb)

    def flush(self):
        pass
