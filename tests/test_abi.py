"""CPU: the C-ABI library loads, exports every symbol declared in include/dpipe.h, and the ctypes layer declares
each of them.  No compute call is made."""
import ctypes

from diffusion_pipe_b200 import _abi, _lib


def test_library_loads_and_reports_version():
    lib = _lib.lib()
    assert lib.dpipe_abi_version() >= 1
    assert isinstance(lib.dpipe_last_error(), bytes)


def test_every_declared_symbol_is_exported():
    lib = _lib.lib()
    syms = _lib.exported_symbols()
    assert len(syms) >= 19
    missing = [s for s in syms if not hasattr(lib, s)]
    assert not missing, f'declared in include/dpipe.h but not exported: {missing}'


def test_ctypes_signatures_cover_the_header():
    known = set(_abi.SIGNATURES) | {'dpipe_last_error', 'dpipe_abi_version', 'dpipe_check_device', 'dpipe_gemm_bf16'}
    assert set(_lib.exported_symbols()) <= known


def test_struct_sizes_match_c_layout():
    # a drifted struct would silently corrupt arguments: pin the sizes the C compiler produces (LP64)
    assert ctypes.sizeof(_lib.QkvEpilogue) == 11 * 8 + 4 * 4 + 4 + 4   # 11 pointers, 4 ints, float, tail padding
    assert ctypes.sizeof(_lib.GemmArgs) % 8 == 0
    assert ctypes.sizeof(_abi.AttnArgs) == 6 * 8 + 4 * 4 + 4 + 4
    assert ctypes.sizeof(_abi.AttnBwdArgs) == 12 * 8 + 4 * 4 + 4 + 4


def test_bad_arguments_fail_loudly_without_a_gpu():
    lib = _lib.lib()
    rc = lib.dpipe_gemm_bf16(None, None)
    assert rc < 0 and b'null' in lib.dpipe_last_error()
    assert lib.dpipe_sched_train(0, 1, 0, None, 0) < 0


def test_struct_sizes_of_the_wan_and_qk_entry_points_match_c_layout():
    # sizes printed by gcc for include/dpipe.h (LP64): dpipe_wan_norm_proj, _fwd_args, _bwd_proj, _bwd_args, dpipe_qk_bwd_args
    assert ctypes.sizeof(_abi.WanNormProj) == 56 and ctypes.sizeof(_abi.WanNormFwdArgs) == 208
    assert ctypes.sizeof(_abi.WanNormBwdProj) == 64 and ctypes.sizeof(_abi.WanNormBwdArgs) == 232
    assert ctypes.sizeof(_abi.QkBwdArgs) == 144


def test_header_compiles_as_plain_c():
    """include/dpipe.h is the boundary a C (not C++) caller binds: it must compile with gcc and agree on the struct sizes"""
    import os
    import shutil
    import subprocess
    import tempfile
    if shutil.which('gcc') is None:
        import pytest
        pytest.skip('gcc not available')
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, 'sz.c')
        with open(src, 'w') as f:
            f.write('#include <stdio.h>\n#include "dpipe.h"\nint main(void){ printf("%zu %zu %zu %zu\\n", sizeof(dpipe_wan_norm_fwd_args), '
                    'sizeof(dpipe_wan_norm_bwd_args), sizeof(dpipe_qk_bwd_args), sizeof(dpipe_instr)); return 0; }\n')
        exe = os.path.join(d, 'sz')
        subprocess.run(['gcc', '-std=c99', '-Wall', '-Werror', '-I', os.path.join(root, 'include'), src, '-o', exe], check=True)
        out = subprocess.run([exe], check=True, capture_output=True, text=True).stdout.split()
    assert [int(x) for x in out] == [ctypes.sizeof(_abi.WanNormFwdArgs), ctypes.sizeof(_abi.WanNormBwdArgs),
                                    ctypes.sizeof(_abi.QkBwdArgs), 12]


def test_entry_points_refuse_bad_arguments_before_any_cuda_call():
    """Wan RMSNorm, LayerNorm, zero-bubble planner and modulation backward: out-of-range shapes fail in the host check,
    so none of these calls (fake pointers) reaches the device"""
    lib = _lib.lib()
    assert lib.dpipe_wan_norm_rope_fwd(None, None) < 0 and b'null' in lib.dpipe_last_error()
    a = _abi.WanNormFwdArgs()
    a.nproj, a.batch, a.seq, a.heads = 1, 1, 8, 57                   # 57 heads: 912-thread CTAs do not fit the register file
    assert lib.dpipe_wan_norm_rope_fwd(ctypes.byref(a), None) < 0 and b'geometry' in lib.dpipe_last_error()
    a.heads = 3                                                     # 384 columns: not a multiple of 256
    assert lib.dpipe_wan_norm_rope_fwd(ctypes.byref(a), None) < 0
    assert lib.dpipe_wan_norm_rope_bwd(None, None) < 0
    # LayerNorm width rules (whole warps, one CTA per row group)
    buf = ctypes.c_void_p(8)
    assert lib.dpipe_ln_modulate_fwd_ex(buf, 100, buf, buf, 0, buf, 100, None, None, 1, 1, 100, 1e-6, 0, None) < 0
    assert b'multiple of 256' in lib.dpipe_last_error()
    assert lib.dpipe_ln_modulate_fwd_ex(buf, 8192, buf, buf, 0, buf, 8192, None, None, 1, 1, 8192, 1e-6, 0, None) < 0
    # zero-bubble planner: weights must be positive and one per stage
    w = (ctypes.c_int * 2)(3, 0)
    assert lib.dpipe_sched_zb_ex(4, 2, 0, 13, 17, 10, 4, w, None, 0) < 0
    assert lib.dpipe_sched_zb_makespan_ex(4, 2, 13, 17, 10, 4, w) < 0
    # the batch-row modulation backward takes 1..8 samples and widths that are multiples of 256 up to 8192
    for B, K in ((9, 5120), (0, 5120), (8, 100), (8, 8448)):
        assert lib.dpipe_mod_bwd(buf, 0, buf, buf, buf, 0, buf, buf, buf, B, 1024, K, None) < 0, (B, K)
        assert b'dpipe_mod_bwd: bad arguments' in lib.dpipe_last_error()


def test_fp8_code_tables_are_torchs_widening_for_all_256_codes():
    """dpipe_fp8_code_table returns the table csrc/fp8_dequant.cu builds in shared memory: every float8_e4m3fn /
    float8_e5m2 code must widen to the bf16 value torch's own cast gives (the reference's autocast widening)"""
    import torch
    lib = _lib.lib()
    for fmt, dt in ((0, torch.float8_e4m3fn), (1, torch.float8_e5m2)):
        out = (ctypes.c_uint16 * 256)()
        assert lib.dpipe_fp8_code_table(fmt, out) == 0
        got = torch.tensor(list(out), dtype=torch.int32).to(torch.int16).view(torch.bfloat16)
        want = torch.arange(256, dtype=torch.uint8).view(dt).to(torch.bfloat16)
        nan = torch.isnan(want.float())
        assert torch.equal(torch.isnan(got.float()), nan)
        assert torch.equal(got.view(torch.int16)[~nan], want.view(torch.int16)[~nan])
        assert int(nan.sum()) == (2 if fmt == 0 else 6)
    assert lib.dpipe_fp8_code_table(2, out) < 0 and lib.dpipe_fp8_code_table(0, None) < 0
    # shape / alignment rules of the kernel entry point are checked before any CUDA call
    buf = ctypes.c_void_p(256)
    assert lib.dpipe_fp8_to_bf16(buf, 64, buf, 64, 4, 60, 0, None) < 0 and b'multiples of 16' in lib.dpipe_last_error()
    assert lib.dpipe_fp8_to_bf16(buf, 64, buf, 60, 4, 64, 0, None) < 0
    assert lib.dpipe_fp8_to_bf16(ctypes.c_void_p(8), 64, buf, 64, 4, 64, 0, None) < 0 and b'aligned' in lib.dpipe_last_error()
    assert lib.dpipe_fp8_to_bf16(buf, 64, buf, 64, 4, 64, 7, None) < 0
    assert lib.dpipe_fp8_to_bf16(buf, 64, buf, 64, 0, 64, 0, None) == 0          # empty matrix: nothing to do


def test_ctypes_argument_lists_match_the_header_prototypes():
    """every prototype of include/dpipe.h against the ctypes declaration that calls it: same number of arguments, and each
    argument in the same class (pointer / 32-bit int / 64-bit int / float / double) — a drifted scalar width would pass
    garbage in a register without any error"""
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, 'include', 'dpipe.h')).read()
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    text = re.sub(r'//[^\n]*', ' ', text)
    protos = re.findall(r'\b(int|long long|const char\s*\*)\s+(dpipe_\w+)\s*\(([^;{}]*?)\)\s*;', text)
    assert len(protos) >= 40

    def cls_of_c(arg):
        a = arg.strip()
        if a in ('void', ''):
            return None
        if '*' in a or a.endswith(']'):
            return 'ptr'
        base = re.sub(r'\b(const|unsigned)\b', '', a).split()
        t = ' '.join(base[:-1]) if len(base) > 1 else base[0]
        return {'int': 'i32', 'int64_t': 'i64', 'uint64_t': 'i64', 'long long': 'i64', 'float': 'f32', 'double': 'f64',
                'size_t': 'i64'}[t]

    def cls_of_ctypes(t):
        if t in (ctypes.c_void_p, ctypes.c_char_p) or hasattr(t, 'contents') or issubclass(t, ctypes._Pointer):
            return 'ptr'
        return {ctypes.c_int: 'i32', ctypes.c_int64: 'i64', ctypes.c_uint64: 'i64', ctypes.c_longlong: 'i64', ctypes.c_float: 'f32',
                ctypes.c_double: 'f64'}[t]
    checked = 0
    for ret, name, args in protos:
        if name not in _abi.SIGNATURES:
            continue
        restype, argtypes = _abi.SIGNATURES[name]
        want = [c for c in (cls_of_c(a) for a in args.split(',')) if c is not None]
        got = [cls_of_ctypes(t) for t in argtypes]
        assert got == want, (name, got, want)
        assert (restype is ctypes.c_longlong) == (ret == 'long long'), name
        checked += 1
    assert checked >= 35, checked


def test_struct_field_offsets_match_the_c_compiler(tmp_path):
    """every field of every argument struct of include/dpipe.h: offsetof() from gcc == the offset ctypes computed, in
    declaration order (equal sizes alone would not notice two swapped fields of the same width... nor would this, but a
    wrong width, a missing field or different padding would shift everything after it)"""
    import os
    import re
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, 'include', 'dpipe.h')).read()
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    pairs = {'dpipe_qkv_epilogue': _lib.QkvEpilogue, 'dpipe_gemm_args': _lib.GemmArgs, 'dpipe_attn_args': _abi.AttnArgs,
             'dpipe_attn_bwd_args': _abi.AttnBwdArgs, 'dpipe_qk_bwd_args': _abi.QkBwdArgs, 'dpipe_wan_norm_proj': _abi.WanNormProj,
             'dpipe_wan_norm_fwd_args': _abi.WanNormFwdArgs, 'dpipe_wan_norm_bwd_proj': _abi.WanNormBwdProj,
             'dpipe_wan_norm_bwd_args': _abi.WanNormBwdArgs}
    fields = {}
    for name in pairs:
        body = re.search(r'typedef struct ' + name + r'\s*\{(.*?)\}\s*' + name + r'\s*;', text, flags=re.S).group(1)
        names = []
        for decl in body.split(';'):
            decl = decl.strip()
            if decl:
                for d in decl.split(','):                                  # `int M, N, K;` declares three fields
                    names.append(re.sub(r'\[.*\]', '', d.split()[-1].lstrip('*')))
        fields[name] = names
    src = '#include <stdio.h>\n#include <stddef.h>\n#include "dpipe.h"\nint main(void){\n'
    for name, names in fields.items():
        for f in names:
            src += f'  printf("{name} {f} %zu\\n", offsetof({name}, {f}));\n'
        src += f'  printf("{name} __size__ %zu\\n", sizeof({name}));\n'
    src += '  return 0; }\n'
    (tmp_path / 'off.c').write_text(src)
    subprocess.run(['gcc', '-std=c99', '-I', os.path.join(root, 'include'), str(tmp_path / 'off.c'), '-o', str(tmp_path / 'off')], check=True)
    out = subprocess.run([str(tmp_path / 'off')], check=True, capture_output=True, text=True).stdout.split('\n')
    c_off = {}
    for line in out:
        if line:
            s, f, o = line.split()
            c_off.setdefault(s, []).append((f, int(o)))
    for name, cls in pairs.items():
        want = [o for f, o in c_off[name] if f != '__size__']
        got = [getattr(cls, fn).offset for fn, _ in cls._fields_]
        assert got == want, (name, [fn for fn, _ in cls._fields_], fields[name], got, want)
        assert ctypes.sizeof(cls) == dict(c_off[name])['__size__'], name


def _tmap_refused(lib):
    """the tensor-map encode refused the call (without a driver it cannot even be looked up: refused all the same)"""
    msg = lib.dpipe_last_error()
    return b'TMA operand' in msg or b'cuTensorMapEncodeTiled entry point not available' in msg


def _gemm_args(epilogue, qkv=None):
    """a GEMM whose A is a TMA operand at address 8: whatever else is wrong, the tensor-map encode refuses the call, so a
    field whose own alignment check were missing could still not reach a launch (every other pointer is aligned)"""
    a = _lib.GemmArgs()
    a.A, a.lda, a.B, a.ldb = 8, 64, 256, 64
    a.M, a.N, a.K = 64, 768, 64
    a.epilogue = epilogue
    a.out, a.ldo, a.out2, a.ldo2 = 256, 768, 256, 768
    a.aux, a.ldaux, a.gate, a.gate_stride = 256, 768, 256, 768
    a.bias = 256
    a.rows_per_batch, a.cta_group = 64, 1
    if qkv is not None:
        a.qkv = ctypes.pointer(qkv)
    return a


def _qkv_args():
    e = _lib.QkvEpilogue()
    for f in ('q', 'k', 'v', 'qhat', 'khat', 'q_norm_w', 'k_norm_w', 'rope_cos', 'rope_sin', 'q_rstd', 'k_rstd'):
        setattr(e, f, 256)
    e.heads, e.seq_total, e.seq_offset, e.n_qkv, e.eps = 2, 64, 0, 768, 1e-6
    return e


def test_gemm_refuses_misaligned_epilogue_pointers_before_any_launch():
    """out, bias, out2 / ldo2, aux / ldaux, gate / gate_stride and the QKV pointers are read or written 16 bytes at a
    time by the epilogue (q_rstd / k_rstd 4 bytes); none is a TMA operand, so the entry point checks them itself"""
    lib = _lib.lib()
    for epi in (_lib.EPI_STORE, _lib.EPI_BIAS_GELU, _lib.EPI_GATE_RES, _lib.EPI_MUL_GELU_GRAD, _lib.EPI_QKV_ROPE):
        a = _gemm_args(epi, _qkv_args())
        assert lib.dpipe_gemm_bf16(ctypes.byref(a), None) < 0 and _tmap_refused(lib), epi
    cases = [(_lib.EPI_STORE, 'out', 264, b'out'), (_lib.EPI_STORE, 'bias', 258, b'bias'),
             (_lib.EPI_BIAS_GELU, 'bias', 264, b'bias'), (_lib.EPI_BIAS_GELU, 'out2', 264, b'out2/ldo2'),
             (_lib.EPI_BIAS_GELU, 'ldo2', 770, b'out2/ldo2'), (_lib.EPI_GATE_RES, 'out2', 260, b'out2/ldo2'),
             (_lib.EPI_GATE_RES, 'aux', 264, b'aux/ldaux'), (_lib.EPI_GATE_RES, 'ldaux', 772, b'aux/ldaux'),
             (_lib.EPI_GATE_RES, 'gate', 264, b'gate/gate_stride'), (_lib.EPI_GATE_RES, 'gate_stride', 769, b'gate/gate_stride'),
             (_lib.EPI_MUL_GELU_GRAD, 'aux', 258, b'aux/ldaux'), (_lib.EPI_MUL_GELU_GRAD, 'ldaux', 770, b'aux/ldaux'),
             (_lib.EPI_QKV_ROPE, 'out2', 264, b'out2/ldo2')]
    for epi, field, value, name in cases:
        a = _gemm_args(epi, _qkv_args())
        setattr(a, field, value)
        assert lib.dpipe_gemm_bf16(ctypes.byref(a), None) < 0, (epi, field)
        assert name + b' misaligned' in lib.dpipe_last_error(), (epi, field, lib.dpipe_last_error())
    for field, value in (('q', 264), ('k', 264), ('v', 264), ('qhat', 264), ('khat', 264), ('q_norm_w', 258),
                         ('k_norm_w', 264), ('rope_cos', 260), ('rope_sin', 264), ('q_rstd', 258), ('k_rstd', 257)):
        e = _qkv_args()
        setattr(e, field, value)
        a = _gemm_args(_lib.EPI_QKV_ROPE, e)
        assert lib.dpipe_gemm_bf16(ctypes.byref(a), None) < 0, field
        assert b'qkv.' + field.encode() + b' misaligned' in lib.dpipe_last_error(), (field, lib.dpipe_last_error())
    # pointers an epilogue does not touch are not checked (here STORE's out2 / aux / gate, and NULL outputs)
    a = _gemm_args(_lib.EPI_STORE)
    a.out2, a.aux, a.gate, a.ldo2 = 258, 258, 258, 3
    assert lib.dpipe_gemm_bf16(ctypes.byref(a), None) < 0 and _tmap_refused(lib)
    e = _qkv_args()
    e.q_rstd = e.k_rstd = e.qhat = e.khat = None
    a = _gemm_args(_lib.EPI_QKV_ROPE, e)
    assert lib.dpipe_gemm_bf16(ctypes.byref(a), None) < 0 and _tmap_refused(lib)


def test_attention_refuses_misaligned_outputs_before_any_launch():
    """attention forward writes o in 4-byte pairs and lse as fp32; the backward reads o / d_o 8 bytes at a time and
    writes dq / dk / dv in pairs, lse / delta as fp32.  q sits at address 8, so the tensor-map encode of q refuses
    every one of these calls even without the checks, and the backward encodes every map before its first launch"""
    lib = _lib.lib()
    a = _abi.AttnArgs()
    a.q, a.k, a.v, a.o, a.lse = 8, 256, 256, 256, 256
    a.ldo, a.batch, a.heads, a.seq_q, a.seq_k, a.scale = 128, 1, 1, 64, 64, 0.1
    assert lib.dpipe_attn_fwd(ctypes.byref(a), None) < 0 and _tmap_refused(lib)
    for field, value in (('o', 258), ('lse', 258)):
        setattr(a, field, value)
        assert lib.dpipe_attn_fwd(ctypes.byref(a), None) < 0, field
        assert f'{field} misaligned'.encode() in lib.dpipe_last_error(), (field, lib.dpipe_last_error())
        setattr(a, field, 256)
    b = _abi.AttnBwdArgs()
    for f in ('k', 'v', 'o', 'd_o', 'lse', 'delta', 'dq', 'dk', 'dv'):
        setattr(b, f, 256)
    b.q, b.ldo, b.lddo, b.batch, b.heads, b.seq_q, b.seq_k, b.scale = 8, 128, 128, 1, 1, 64, 64, 0.1
    assert lib.dpipe_attn_bwd(ctypes.byref(b), None) < 0 and _tmap_refused(lib)
    for field, value in (('o', 260), ('d_o', 260), ('dq', 258), ('dk', 258), ('dv', 258), ('lse', 258), ('delta', 257)):
        setattr(b, field, value)
        assert lib.dpipe_attn_bwd(ctypes.byref(b), None) < 0, field
        assert f'{field} misaligned'.encode() in lib.dpipe_last_error(), (field, lib.dpipe_last_error())
        setattr(b, field, 256)
