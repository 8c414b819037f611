"""ctypes structures and signatures for the C-ABI entry points beyond the GEMM (kept in one place so that the
CPU-side test can check every symbol of include/dpipe.h is both exported and declared)."""
import ctypes

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_int64 = ctypes.c_int64
c_float = ctypes.c_float

SIGNATURES = {}


def declare(l):
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(l, name, None)
        if fn is None:
            continue
        fn.restype = restype
        fn.argtypes = argtypes


class AttnArgs(ctypes.Structure):
    _fields_ = [
        ('q', c_void_p), ('k', c_void_p), ('v', c_void_p),
        ('o', c_void_p), ('ldo', c_int64),
        ('lse', c_void_p),
        ('batch', c_int), ('heads', c_int), ('seq_q', c_int), ('seq_k', c_int),
        ('scale', c_float),
    ]


class AttnBwdArgs(ctypes.Structure):
    _fields_ = [
        ('q', c_void_p), ('k', c_void_p), ('v', c_void_p),
        ('o', c_void_p), ('ldo', c_int64),
        ('d_o', c_void_p), ('lddo', c_int64),
        ('lse', c_void_p), ('delta', c_void_p),
        ('dq', c_void_p), ('dk', c_void_p), ('dv', c_void_p),
        ('batch', c_int), ('heads', c_int), ('seq_q', c_int), ('seq_k', c_int),
        ('scale', c_float),
    ]


class QkBwdArgs(ctypes.Structure):
    _fields_ = [
        ('dq', c_void_p), ('dk', c_void_p), ('dv', c_void_p),
        ('qhat', c_void_p), ('khat', c_void_p),
        ('q_rstd', c_void_p), ('k_rstd', c_void_p),
        ('q_norm_w', c_void_p), ('k_norm_w', c_void_p),
        ('rope_cos', c_void_p), ('rope_sin', c_void_p),
        ('dqkv', c_void_p), ('ld', c_int64),
        ('dbias', c_void_p), ('dw', c_void_p),
        ('batch', c_int), ('heads', c_int), ('seq_total', c_int), ('seq_offset', c_int), ('rows_per_batch', c_int),
    ]


class WanNormProj(ctypes.Structure):
    _fields_ = [('src', c_void_p), ('ld', c_int64), ('weight', c_void_p), ('dst', c_void_p), ('xhat', c_void_p),
                ('rstd', c_void_p), ('rope', c_int)]


class WanNormFwdArgs(ctypes.Structure):
    _fields_ = [('proj', WanNormProj * 3), ('nproj', c_int), ('cos', c_void_p), ('sin', c_void_p),
                ('batch', c_int), ('seq', c_int), ('heads', c_int), ('eps', c_float)]


class WanNormBwdProj(ctypes.Structure):
    _fields_ = [('dy', c_void_p), ('xhat', c_void_p), ('rstd', c_void_p), ('weight', c_void_p), ('dx', c_void_p),
                ('ld', c_int64), ('dw_partials', c_void_p), ('rope', c_int)]


class WanNormBwdArgs(ctypes.Structure):
    _fields_ = [('proj', WanNormBwdProj * 3), ('nproj', c_int), ('cos', c_void_p), ('sin', c_void_p),
                ('batch', c_int), ('seq', c_int), ('heads', c_int)]


SIGNATURES['dpipe_wan_norm_rope_fwd'] = (c_int, [ctypes.POINTER(WanNormFwdArgs), c_void_p])
SIGNATURES['dpipe_wan_norm_rope_bwd'] = (c_int, [ctypes.POINTER(WanNormBwdArgs), c_void_p])
SIGNATURES['dpipe_wan_norm_rows'] = (c_int, [])
SIGNATURES['dpipe_attn_fwd'] = (c_int, [ctypes.POINTER(AttnArgs), c_void_p])
SIGNATURES['dpipe_attn_bwd'] = (c_int, [ctypes.POINTER(AttnBwdArgs), c_void_p])
SIGNATURES['dpipe_row_chunk'] = (c_int, [])
SIGNATURES['dpipe_ln_modulate_fwd'] = (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p, c_int64,
                                               c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p])
SIGNATURES['dpipe_ln_modulate_bwd'] = (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p,
                                               c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int, c_int,
                                               c_int, c_void_p])
SIGNATURES['dpipe_ln_modulate_fwd_ex'] = (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_void_p, c_int64,
                                                  c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_int, c_void_p])
SIGNATURES['dpipe_ln_modulate_bwd_ex'] = (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p,
                                                  c_void_p, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int, c_int,
                                                  c_int, c_int, c_void_p])
SIGNATURES['dpipe_gate_bwd'] = (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64,
                                        c_void_p, c_int, c_int, c_int, c_void_p])
SIGNATURES['dpipe_colreduce_finish'] = (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int64, c_void_p,
                                                c_int64, c_void_p, c_void_p, c_void_p])
SIGNATURES['dpipe_colsum_chunks'] = (c_int, [c_int])
SIGNATURES['dpipe_colsum'] = (c_int, [c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p, c_void_p])
SIGNATURES['dpipe_qknorm_rope_bwd'] = (c_int, [ctypes.POINTER(QkBwdArgs), c_void_p])
SIGNATURES['dpipe_sched_num_pipe_buffers'] = (c_int, [c_int, c_int, c_int])
SIGNATURES['dpipe_sched_train'] = (c_int, [c_int, c_int, c_int, c_void_p, c_int])
SIGNATURES['dpipe_sched_infer'] = (c_int, [c_int, c_int, c_int, c_void_p, c_int])
SIGNATURES['dpipe_sched_zb'] = (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int])
SIGNATURES['dpipe_sched_zb_makespan'] = (ctypes.c_longlong, [c_int, c_int, c_int, c_int, c_int, c_int])
SIGNATURES['dpipe_sched_zb_ex'] = (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int])
SIGNATURES['dpipe_sched_zb_makespan_ex'] = (ctypes.c_longlong, [c_int, c_int, c_int, c_int, c_int, c_int, c_void_p])
SIGNATURES['dpipe_partition_balanced'] = (c_int, [c_void_p, c_int, c_int, c_void_p])
SIGNATURES['dpipe_ipc_alloc'] = (c_int, [c_int64, ctypes.POINTER(c_void_p), c_void_p])
SIGNATURES['dpipe_ipc_open'] = (c_int, [c_void_p, ctypes.POINTER(c_void_p)])
SIGNATURES['dpipe_ipc_close'] = (c_int, [c_void_p])
SIGNATURES['dpipe_ipc_free'] = (c_int, [c_void_p])
SIGNATURES['dpipe_peer_copy'] = (c_int, [c_void_p, c_int, c_void_p, c_int, c_int64, c_void_p])
SIGNATURES['dpipe_flag_write'] = (c_int, [c_void_p, ctypes.c_uint64, c_void_p])
SIGNATURES['dpipe_flag_wait_geq'] = (c_int, [c_void_p, ctypes.c_uint64, ctypes.c_double, c_void_p])
SIGNATURES['dpipe_mod_fwd'] = (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p])
SIGNATURES['dpipe_mod_bwd_chunks'] = (c_int, [c_int])
SIGNATURES['dpipe_mod_bwd'] = (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                        c_int, c_int, c_int, c_void_p])
SIGNATURES['dpipe_mse_loss'] =(c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p])
SIGNATURES['dpipe_fp8_to_bf16'] = (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p])
SIGNATURES['dpipe_fp8_code_table'] = (c_int, [c_int, c_void_p])
SIGNATURES['dpipe_grad_sumsq_blocks'] = (c_int, [])
SIGNATURES['dpipe_grad_sumsq'] = (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_void_p, c_void_p])
SIGNATURES['dpipe_grad_scale'] = (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p])
SIGNATURES['dpipe_adamw_step'] = (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_float,
                                          c_float, c_float, c_float, c_float, c_float, c_void_p])
SIGNATURES['dpipe_automagic_scratch_doubles'] = (c_int, [c_void_p, c_int, ctypes.POINTER(c_int64)])
SIGNATURES['dpipe_automagic_stats'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int64, c_void_p])
SIGNATURES['dpipe_automagic_apply'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p])
SIGNATURES['dpipe_prodigy_scratch_doubles'] = (c_int, [c_void_p, c_int, ctypes.POINTER(c_int64)])
SIGNATURES['dpipe_prodigy_stats'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_void_p])
SIGNATURES['dpipe_prodigy_apply'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p])
SIGNATURES['dpipe_adamw8bit_step'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p])
SIGNATURES['dpipe_came_scratch_doubles'] = (c_int, [c_void_p, c_int, ctypes.POINTER(c_int64)])
SIGNATURES['dpipe_came_step'] = (c_int, [c_void_p, c_int, ctypes.c_double, c_void_p, c_int64, c_void_p])
SIGNATURES['dpipe_noise_pack'] = (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int64, c_int, c_int,
                                          c_int, c_void_p])
SIGNATURES['dpipe_exec_create'] = (c_int, [c_int, c_int, ctypes.c_double, ctypes.POINTER(c_void_p)])
SIGNATURES['dpipe_exec_destroy'] = (c_int, [c_void_p])
SIGNATURES['dpipe_exec_copy_stream'] = (c_void_p, [c_void_p])
SIGNATURES['dpipe_exec_bind'] = (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_int64, c_int64, c_int])
SIGNATURES['dpipe_exec_set_layout'] = (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p])
SIGNATURES['dpipe_exec_forget_layouts'] = (c_int, [c_void_p])
SIGNATURES['dpipe_exec_load_plan'] = (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int])
SIGNATURES['dpipe_exec_stage_send'] = (c_int, [c_void_p, c_int, c_int, c_int, c_void_p])
SIGNATURES['dpipe_exec_recv_base'] = (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(c_void_p)])
SIGNATURES['dpipe_exec_next'] = (c_int, [c_void_p, c_void_p, c_void_p])


class AutomagicTensor(ctypes.Structure):
    _fields_ = [('p', c_void_p), ('g', c_void_p), ('row', c_void_p), ('col', c_void_p), ('v', c_void_p),
                ('code', c_void_p), ('pol', c_void_p), ('shift', c_void_p), ('scale', c_void_p), ('avg_lr', c_void_p),
                ('ws', c_void_p), ('numel', c_int64), ('L', c_int64), ('R', c_int64), ('C', c_int64),
                ('dtype', c_int), ('flags', c_int)]


class AutomagicScalars(ctypes.Structure):
    _fields_ = [('beta2', ctypes.c_double), ('eps', ctypes.c_double), ('lr_bump', ctypes.c_double),
                ('min_lr', ctypes.c_double), ('max_lr', ctypes.c_double), ('clip_threshold', ctypes.c_double),
                ('weight_decay', ctypes.c_double)]


class ProdigyTensor(ctypes.Structure):
    _fields_ = [('p', c_void_p), ('g', c_void_p), ('p0', c_void_p), ('s', c_void_p), ('m', c_void_p), ('v', c_void_p),
                ('numel', c_int64), ('weight_decay', ctypes.c_double), ('eps', ctypes.c_double), ('dtype', c_int),
                ('fixed_decay', c_int)]


class ProdigyScalars(ctypes.Structure):
    _fields_ = [('lr', ctypes.c_double), ('beta1', ctypes.c_double), ('beta2', ctypes.c_double),
                ('beta3', ctypes.c_double), ('d0', ctypes.c_double), ('d_coef', ctypes.c_double),
                ('growth_rate', ctypes.c_double), ('bias_correction', c_int), ('safeguard_warmup', c_int)]


# slots of the Prodigy device scalar block (include/dpipe.h DPIPE_PRODIGY_*)
PRODIGY_SLOTS = {'d': 0, 'd_max': 1, 'd_hat': 2, 'd_numerator': 3, 'd_denom': 4, 'step': 5, 'd_lr': 6, 'skip': 7}
PRODIGY_STATE_DOUBLES = 8


class Adamw8bitTensor(ctypes.Structure):
    _fields_ = [('p', c_void_p), ('g', c_void_p), ('state1', c_void_p), ('state2', c_void_p), ('absmax1', c_void_p),
                ('absmax2', c_void_p), ('numel', c_int64), ('step_size', c_float), ('beta1', c_float),
                ('beta2', c_float), ('eps_c2', c_float), ('decay', c_float), ('dtype', c_int)]


class CameTensor(ctypes.Structure):
    _fields_ = [('p', c_void_p), ('g', c_void_p), ('m', c_void_p), ('row', c_void_p), ('col', c_void_p),
                ('res_row', c_void_p), ('res_col', c_void_p), ('v', c_void_p), ('fac', c_void_p), ('sums', c_void_p),
                ('numel', c_int64), ('L', c_int64), ('R', c_int64), ('C', c_int64), ('lr', ctypes.c_double),
                ('weight_decay', ctypes.c_double), ('beta1', ctypes.c_double), ('beta2', ctypes.c_double),
                ('beta3', ctypes.c_double), ('eps1', ctypes.c_double), ('eps2', ctypes.c_double), ('dtype', c_int),
                ('factored', c_int), ('fixed_decay', c_int)]
