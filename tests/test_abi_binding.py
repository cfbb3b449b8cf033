"""CPU: the ctypes binding that _lib derives from include/ptb_b200.h on import (no library needed).  Pins the derived signatures of
declarations that exercise every type rule, the two struct layouts, the values ops and assigners take from the header's #defines,
and the parser's refusal of what it does not know."""
import ctypes

import pytest
import torch

from pointtinybenchmark_b200 import _lib, assigners, ops

I, I64, U64, F, D, P = ctypes.c_int, ctypes.c_int64, ctypes.c_uint64, ctypes.c_float, ctypes.c_double, ctypes.c_void_p

SIGNATURES = {
    'ptb_last_error': (ctypes.c_char_p, []),                         # const char* return, (void)
    'ptb_cpr_refine': (I, [P, P, P, I, I, I, I, P, P, P, P, P, P, P, _lib.RefineCfg, P, P, P, P, P, P]),     # struct by value
    'ptb_p2p_decode_topk_levels': (I, [P, P, I, P, P, I, I, I, P, F, P, P, I, P, P, P, P, U64, P]),            # const float* const*
    'ptb_roi_align_bwd': (I, [P, P, P, I, I, I, P, P, I, I, I, P, P]),                                         # float* const*
    'ptb_p2p_cost_matrix_terms': (I, [P, P, I, P, I, I, P, P, I, P, I, F, F, P, P, U64, P]),                   # const ptb_match_cost*
    'ptb_ghmc_bin_weights': (I, [P, P, P, I, I64, I, P, I, D, P, P, P, P, P]),                                 # double, int64_t
    'ptb_rpn_proposals_workspace': (U64, [P, I, I, I, I, I]),                                                  # uint64_t return
}


@pytest.mark.parametrize('name', list(SIGNATURES))
def test_derived_signature(name):
    assert _lib.SIGNATURES[name] == SIGNATURES[name]


def test_struct_layouts():
    assert _lib.RefineCfg._fields_ == [('merge_th', F), ('gt_alpha', F), ('refine_th', F), ('flags', ctypes.c_int32)]
    assert ctypes.sizeof(_lib.RefineCfg) == 16
    assert _lib.MatchCost._fields_ == [('kind', ctypes.c_int32), ('weight', F), ('alpha', F), ('gamma', F), ('eps', F),
                                       ('p', ctypes.c_int32), ('norm_with_img_wh', ctypes.c_int32)]
    assert ctypes.sizeof(_lib.MatchCost) == 28
    assert ops.RefineCfg is _lib.RefineCfg


def test_constants_from_the_header():
    assert _lib.DEFINES['PTB_ABI_VERSION'] == 2
    assert ops.GHM_MAX_BINS == 256
    assert (ops.RPN_LOSS_L1, ops.RPN_LOSS_SMOOTH_L1) == (0, 1)
    assert (ops.ROI_MAX_LEVELS, ops.RPN_MAX_LEVELS, ops.BATCHED_NMS_MAX_ROWS) == (4, 8, 65536)
    assert ops.HALF_DTYPES == {torch.float16: 1, torch.bfloat16: 2}
    assert ops.LOSS_KINDS == {'gfocal_loss': 0, 'binary_cross_entropy': 1}
    assert ops.MATCH_COST_KINDS == {'FocalLossCost': 0, 'ClassificationCostV2_sigmoid': 1, 'ClassificationCostV2_softmax': 2,
                                    'ZeroCost': 3, 'DisCostV2': 4}
    assert assigners.MAX_MATCH_COST_TERMS == 8


def test_parse_header_on_a_string():
    sigs, structs, defines = _lib.parse_header(
        '/* a comment; with a semicolon */\n#define PTB_A 3\n#define PTB_NEG -1\n#ifdef __cplusplus\nextern "C" {\n#endif\n'
        'typedef struct {\n  int32_t k;  /* kind */\n  float w, v;\n} ptb_two_terms;\n'
        'int ptb_f(const ptb_two_terms* t, ptb_two_terms by_value, int64_t n,\n          const float* const* maps, void* stream);\n'
        '#ifdef __cplusplus\n}\n#endif\n')
    assert defines == {'PTB_A': 3, 'PTB_NEG': -1}
    s = structs['ptb_two_terms']
    assert s.__name__ == 'TwoTerms' and s._fields_ == [('k', I), ('w', F), ('v', F)]
    assert sigs == {'ptb_f': (I, [P, s, I64, P, P])}


@pytest.mark.parametrize('text, what', [
    ('int ptb_x(size_t n, void* stream);', "unknown type 'size_t'"),
    ('int ptb_x(unsigned n);', "unknown type 'unsigned'"),
    ('void ptb_x(int n);', "unknown type 'void'"),
    ('typedef struct { float a; } ptb_s;\nptb_s ptb_x(void);', "unknown type 'ptb_s'"),
    ('int ptb_x(int, void* stream);', 'unnamed parameter'),
    ('int ptb_x[4];', 'not a ptb_\\* prototype'),
])
def test_parser_refuses_what_it_does_not_know(text, what):
    with pytest.raises(ValueError, match=what) as e:
        _lib.parse_header(text)
    assert 'ptb_x' in str(e.value)


def test_parser_refuses_a_struct_member_it_does_not_know():
    with pytest.raises(ValueError, match='ptb_s'):
        _lib.parse_header('typedef struct { float a[4]; } ptb_s;')
