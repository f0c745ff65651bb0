"""CPU tests of the C-ABI boundary: the library loads without a GPU, exports every symbol include/ttsb.h declares,
validates arguments and reports errors through ttsb_last_error (no compute calls here)."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope='module')
def cdll():
    from transformertts_b200 import build, lib
    build.build(verbose=False)
    return lib.load()


def test_header_symbols_are_all_exported(cdll):
    header = (ROOT / 'include' / 'ttsb.h').read_text()
    names = set(re.findall(r'\b(ttsb_[a-z0-9_]+)\s*\(', header))
    names -= {'ttsb_gemm_args', 'ttsb_mha_args'}
    assert len(names) >= 18
    for n in sorted(names):
        assert hasattr(cdll, n), f'{n} declared in include/ttsb.h but not exported by libttsb.so'
    from transformertts_b200 import lib
    assert set(lib.EXPORTS) == names


def test_abi_version_5_and_error_text(cdll):
    assert cdll.ttsb_abi_version() == 5
    rc = cdll.ttsb_linear_fwd(None, None)
    assert rc == -1
    assert b'NULL' in cdll.ttsb_last_error()


def _header_structs(header: str) -> dict:
    """{struct name: [(field, C type, array length)]} of every `typedef struct name { ... } name;` in the header."""
    macros = {m: int(v) for m, v in re.findall(r'#define (\w+) (\d+)', header)}
    structs = {}
    for name, body in re.findall(r'typedef struct (\w+) \{(.*?)\} \1;', header, re.S):
        fields = []
        for decl in re.sub(r'/\*.*?\*/', '', body, flags=re.S).split(';'):
            if not decl.strip():
                continue
            ctype, first = re.match(r'\s*(.*?[\s*])(\w+(?:\[\w+\])?)$', decl.split(',')[0].rstrip()).groups()
            for part in [first] + [d.strip() for d in decl.split(',')[1:]]:
                fname, n = re.fullmatch(r'(\w+)(?:\[(\w+)\])?', part).groups()
                fields.append((fname, ctype.strip(), None if n is None else int(macros.get(n, n))))
        structs[name] = fields
    return structs


def _mirrors(lib) -> dict:
    """{header struct name: its ctypes mirror in lib.py}"""
    return {'ttsb_pack_desc': lib.PackDesc, 'ttsb_gemm_args': lib.GemmArgs, 'ttsb_mha_args': lib.MhaArgs,
            'ttsb_decode_attn_args': lib.DecodeAttnArgs, 'ttsb_bgemm_args': lib.BgemmArgs, 'ttsb_wgrad_args': lib.WgradArgs,
            'ttsb_conv1d_ex_args': lib.Conv1dExArgs}


def test_struct_layout_matches_header():
    """Every ctypes mirror in lib.py against its typedef struct: field names and order, C types, array lengths, offsets and
    size; and the constants lib.py mirrors of the header's #defines."""
    from transformertts_b200 import lib
    header = (ROOT / 'include' / 'ttsb.h').read_text()
    structs = _header_structs(header)
    mirrors = _mirrors(lib)
    assert set(structs) == set(mirrors)
    assert set(mirrors.values()) == {v for v in vars(lib).values() if isinstance(v, type) and issubclass(v, C.Structure)}
    scalars = {'int': C.c_int, 'int64_t': C.c_int64, 'long long': C.c_longlong, 'uint32_t': C.c_uint32, 'float': C.c_float}
    for struct, cls in mirrors.items():
        fields = structs[struct]
        assert [f[0] for f in fields] == [f[0] for f in cls._fields_], struct
        offset = align = 0
        for (name, ctype, n), (_, ptype) in zip(fields, cls._fields_):
            base = C.c_void_p if ctype.endswith('*') else scalars[ctype]
            if n is None:
                assert ptype is base, (struct, name)
            else:
                assert issubclass(ptype, C.Array) and ptype._type_ is base and ptype._length_ == n, (struct, name)
            size = C.sizeof(base)
            offset = -(-offset // size) * size
            assert getattr(cls, name).offset == offset, (struct, name)
            offset += size * (n or 1)
            align = max(align, size)
        assert C.sizeof(cls) == -(-offset // align) * align, struct
    for macro, value in (('TTSB_PREC_BF16', lib.PREC_BF16), ('TTSB_PREC_BF16X3', lib.PREC_BF16X3), ('TTSB_PREC_FP16', lib.PREC_FP16),
                         ('TTSB_IMPL_TCGEN05', lib.IMPL_TCGEN05), ('TTSB_IMPL_SIMT', lib.IMPL_SIMT),
                         ('TTSB_HALO_NONE', lib.HALO_NONE), ('TTSB_HALO_REFLECT', lib.HALO_REFLECT), ('TTSB_HALO_ZERO', lib.HALO_ZERO),
                         ('TTSB_CONV1D_EX_MAX_TAPS', lib.CONV1D_EX_MAX_TAPS), ('TTSB_CONV1D_EX_MAX_HALO', lib.CONV1D_EX_MAX_HALO),
                         ('TTSB_CONV1D_SUM_NONE', lib.SUM_NONE), ('TTSB_CONV1D_SUM_WRITE', lib.SUM_WRITE),
                         ('TTSB_CONV1D_SUM_ADD', lib.SUM_ADD), ('TTSB_CONV1D_SUM_FINISH', lib.SUM_FINISH)):
        assert re.search(r'#define %s (\d+)' % macro, header).group(1) == str(value), macro


def _header_prototypes(header: str) -> dict:
    """{function name: (return type, [parameter types])} of every prototype in the header, types as written."""
    protos = {}
    for ret, name, params in re.findall(r'^[ \t]*((?:const\s+)?\w+[\s*]*?)\s*\b(ttsb_\w+)\s*\(([^)]*)\)\s*;',
                                        re.sub(r'/\*.*?\*/', '', header, flags=re.S), re.M):
        params = [] if params.strip() == 'void' else [re.fullmatch(r'\s*(.*?)\s*\w+\s*', p, re.S).group(1) for p in params.split(',')]
        protos[name] = (ret, params)
    return protos


def test_signatures_match_header(cdll):
    """lib.SIGNATURES against every prototype of include/ttsb.h: the same names, and for each the return type and the type of
    every parameter in order.  A pointer maps to c_void_p, except a pointer to a ttsb_*_args struct, which maps to a pointer
    to its ctypes mirror.  load() declares every row, and no other module declares libttsb signatures."""
    from transformertts_b200 import lib
    protos = _header_prototypes((ROOT / 'include' / 'ttsb.h').read_text())
    assert len(protos) >= 100
    assert set(lib.SIGNATURES) == set(protos)
    mirrors = _mirrors(lib)
    scalars = {'int': C.c_int, 'int32_t': C.c_int, 'int64_t': C.c_int64, 'uint32_t': C.c_uint32, 'float': C.c_float,
               'double': C.c_double}

    def ctype(decl: str):
        base = re.sub(r'\bconst\b', '', decl).replace('*', ' ').strip()
        if decl.count('*') == 1 and re.fullmatch(r'ttsb_\w+_args', base):
            return C.POINTER(mirrors[base])
        return C.c_void_p if '*' in decl else scalars[base]

    for name, (ret, params) in protos.items():
        restype, argtypes = lib.SIGNATURES[name]
        assert restype is {'const char*': C.c_char_p, 'void': None, **scalars}[ret], (name, ret)
        assert len(argtypes) == len(params), name
        for i, (have, decl) in enumerate(zip(argtypes, params)):
            assert have is ctype(decl), (name, i, decl)
        assert getattr(cdll, name).restype is restype and list(getattr(cdll, name).argtypes) == argtypes, name
    for f in ROOT.rglob('*.py'):
        if f != ROOT / 'transformertts_b200' / 'lib.py' and '_ref' not in f.parts:
            assert not re.search(r'\.(argtypes|restype)\s*=', f.read_text()), f


def test_argument_validation_without_gpu(cdll):
    from transformertts_b200 import lib
    a = lib.GemmArgs()
    a.B, a.T, a.N, a.block_n, a.num_segments = 1, 8, 64, 48 + 1, 1
    assert cdll.ttsb_linear_fwd(C.byref(a), None) == -1
    assert b'block_n' in cdll.ttsb_last_error()
    m = lib.MhaArgs()
    assert cdll.ttsb_mha_fwd(C.byref(m), None) == -1
    # ttsb_mha_fwd refuses column layouts whose H*dh columns leave their row, and a weights row outside the batch, before
    # any launch (fake non-null pointers: nothing may be read or written)
    p = C.c_void_p(256)

    def mha(cross=False, **kw):
        a = lib.MhaArgs()
        a.B, a.T, a.H, a.dh = 2, 70, 2, 64
        a.qk_hi, a.qk_lo, a.kv_len, a.out_hi, a.out_lo = p, p, p, p, p
        a.ld_qk, a.q_col0, a.k_col0, a.v_col0, a.ld_out = 3 * 128, 0, 128, 256, 128
        a.precision, a.impl, a.full_queries = lib.PREC_BF16, lib.IMPL_TCGEN05, int(cross)
        if cross:
            a.ld_qk, a.kv_hi, a.kv_lo, a.ld_kv, a.Tk, a.k_col0, a.v_col0 = 128, p, p, 256, 33, 0, 128
        for k, v in kw.items():
            setattr(a, k, v)
        return cdll.ttsb_mha_fwd(C.byref(a), None)

    for impl in (lib.IMPL_TCGEN05, lib.IMPL_SIMT):
        for bad in ({'q_col0': -8}, {'k_col0': -8}, {'v_col0': -128}, {'q_col0': 264}, {'k_col0': 264}, {'v_col0': 264},
                    {'ld_qk': 376}, {'ld_out': 112}, {'dh': 0}, {'weights_out': p, 'weights_batch_index': 2},
                    {'weights_out': p, 'weights_batch_index': -1}, {'cross': True, 'k_col0': 136},
                    {'cross': True, 'v_col0': 136}, {'cross': True, 'ld_kv': 248}, {'cross': True, 'q_col0': 8},
                    {'cross': True, 'ld_out': 64}):
            assert mha(impl=impl, **bad) == -1, bad
            assert b'ttsb_mha_fwd' in cdll.ttsb_last_error(), bad
    assert cdll.ttsb_stft_mel_log(None, 1, 1000, None, None, 80, 0, None, None) == -1
    # the fused log-mel reads its band table on the host and refuses bad arguments, naming them, before any CUDA call
    band = (C.c_int32 * 256)(*[0, 513] * 128)
    for args, what in (((1, 512, 80, 0), b'n_samples'), ((0, 1000, 80, 0), b'n_clips'), ((1, 1000, 0, 0), b'n_mels'),
                       ((1, 1000, 129, 0), b'n_mels'), ((1, 1000, 80, 2), b'normalizer')):
        n_clips, n_samples, n_mels, norm = args
        assert cdll.ttsb_stft_mel_log(p, n_clips, n_samples, p, band, n_mels, norm, p, None) == -1, args
        assert what in cdll.ttsb_last_error(), args
    for row in ((-1, 4), (5, 4), (0, 514)):
        bad = (C.c_int32 * 4)(0, 513, *row)
        assert cdll.ttsb_stft_mel_log(p, 1, 1000, p, bad, 2, 0, p, None) == -1, row
        assert b'band row 1' in cdll.ttsb_last_error(), row
    assert cdll.ttsb_durations_to_int(None, C.c_float(1.0), None, None, 1, 1, None, None, None) == -1
    # the training attention kernels: the support query is pure host logic; bad arguments are refused before any CUDA call
    assert cdll.ttsb_attn_probs_supported(128, 1008) == 1 and cdll.ttsb_attn_probs_supported(64, 48) == 1
    assert cdll.ttsb_attn_probs_supported(192, 208) == 1
    assert cdll.ttsb_attn_probs_supported(256, 1008) == 0      # head sizes above 192 take the two-kernel path
    assert cdll.ttsb_attn_probs_supported(96, 1008) == 0 and cdll.ttsb_attn_probs_supported(128, 1001) == 0
    assert cdll.ttsb_attn_probs_fwd(None, 768, 0, 256, 1, 2, 100, 128, None, C.c_float(0.1), C.c_float(0.1), 0, 0, None, None, 112, None) == -1
    assert b'ttsb_attn_probs_fwd' in cdll.ttsb_last_error()
    assert cdll.ttsb_attn_ds_bwd(None, 256, 0, None, 768, 512, 1, 2, 100, 128, None, None, None, C.c_float(0.1), C.c_float(0.1), 0, 0, None, 112, None) == -1
    assert b'ttsb_attn_ds_bwd' in cdll.ttsb_last_error()
    # the length-regulator backward reads rows as float4 and scans a row's durations in shared memory: widths that are not
    # a multiple of 4 and more than 12000 phonemes are refused (fake non-null pointers: nothing is launched)
    p = C.c_void_p(16)
    assert cdll.ttsb_expand_bwd(p, p, 1, 8, 16, 6, p, None) == -1
    assert b'ttsb_expand_bwd: need d % 4 == 0' in cdll.ttsb_last_error()
    assert cdll.ttsb_expand_bwd(p, p, 1, 12001, 16, 256, p, None) == -1
    assert b'ttsb_expand_bwd: Tp too large' in cdll.ttsb_last_error()


def test_product_package_never_imports_the_oracle():
    """The oracle is test infrastructure: the product path must not route through it."""
    for f in (ROOT / 'transformertts_b200').rglob('*.py'):
        src = f.read_text()
        assert 'import oracle' not in src and 'from oracle' not in src, f
