"""Every kernel behind the GEMM's row-mapped epilogues, the CUDA-core LayerNorm and the token placement, each with
the debug-hook arguments that select it.

tests/test_kernel_matrix_cpu.py ties these tables to the sources: a new k_gemm_tc instantiation, LayerNorm kernel or
rows_to_split kernel without a row here fails on the CPU.  tests/test_gpu_row_maps.py runs every row, checks under
torch.profiler that exactly the listed kernel launched, and compares its output with float64.
"""

# k_gemm_tc<BN, EPI, ACT> (gemm_tc.cu): the epilogue enum and the activations (common.cuh ActKind)
EPI = {"EPI_FAST": 0, "EPI_LN": 1, "EPI_GENERIC": 2, "EPI_RES": 3, "EPI_F32": 4}
ACT = {"ACT_NONE": 0, "ACT_GELU": 1, "ACT_RELU": 2, "ACT_SILU": 3, "ACT_QUICKGELU": 4, "ACT_LEAKY": 5}
FAST, LN, GENERIC, RES, F32 = (EPI[k] for k in ("EPI_FAST", "EPI_LN", "EPI_GENERIC", "EPI_RES", "EPI_F32"))
NONE, GELU, RELU, SILU, QUICKGELU, LEAKY = range(6)

# tc_gemm's selection, in its order:
#   a LayerNorm (gamma)                               -> EPI_LN, BN 256 (N = 256)
#   a residual R without gamma (fp32 out, N even)     -> EPI_RES
#   split16 out, identity map, no table / zeroing, bias, N % BN == 0, act in {none, GELU, quick-GELU, LeakyReLU}
#                                                     -> EPI_FAST<act> (k_proj_tc instead when K == 256 from one source)
#   vec_f32, fp32 out, identity map, N and ldc even, 8-byte aligned out, act in {none, LeakyReLU}
#                                                     -> EPI_F32<act>
#   anything else                                     -> EPI_GENERIC
# BN = 256 when N % 256 == 0, else 128.  Ragged N = 263 for the generic epilogue; the residual epilogue needs an even
# N, so its ragged row takes 262.  Every row runs at K in GEMM_KS (none of them 256, which would send a fast row to
# k_proj_tc) with the A columns from one source and from two.
GEMM_TC = [
    # ((BN, EPI, ACT), hook arguments)
    ((256, FAST, NONE), dict(N=512, split_out=True, act=NONE)),
    ((128, FAST, NONE), dict(N=384, split_out=True, act=NONE)),
    ((256, FAST, GELU), dict(N=512, split_out=True, act=GELU)),
    ((128, FAST, GELU), dict(N=384, split_out=True, act=GELU)),
    ((256, FAST, QUICKGELU), dict(N=512, split_out=True, act=QUICKGELU)),
    ((128, FAST, QUICKGELU), dict(N=384, split_out=True, act=QUICKGELU)),
    ((256, FAST, LEAKY), dict(N=512, split_out=True, act=LEAKY)),
    ((128, FAST, LEAKY), dict(N=384, split_out=True, act=LEAKY)),
    ((256, GENERIC, NONE), dict(N=512, split_out=True, act=RELU)),          # ReLU is not a fast activation
    ((128, GENERIC, NONE), dict(N=263, split_out=True, act=SILU, out_cols=264)),   # ragged N inside a wider buffer
    ((256, RES, NONE), dict(N=256, residual=True)),
    ((128, RES, NONE), dict(N=262, residual=True)),
    ((256, LN, NONE), dict(N=256, layer_norm=True)),
    ((256, F32, NONE), dict(N=512, vec_f32=True, act=NONE)),
    ((128, F32, NONE), dict(N=384, vec_f32=True, act=NONE)),
    ((256, F32, LEAKY), dict(N=512, vec_f32=True, act=LEAKY)),
    ((128, F32, LEAKY), dict(N=384, vec_f32=True, act=LEAKY)),
]
# one k-block; five (the ring wraps at an odd count for the 2-stage BN = 256 and the 3-stage BN = 128 ring); 17
GEMM_KS = (64, 320, 1088)


def gemm_tc_name(key):
    """The demangled name torch.profiler reports for k_gemm_tc<BN, EPI, ACT> (EPI and ACT are int parameters)."""
    return "k_gemm_tc<%d, %d, %d>" % key


# simt_ln's choice: the 128-bit kernels for d = 256 / 512 when every row it touches is 16-byte aligned, else one
# column per lane in 8 / 16 / 32 columns per lane.  "aligned" False: the output's leading dimension is d + 1.
LN_CASES = [
    # (d, aligned, kernel)
    (64, True, "k_ln<8>"),
    (256, True, "k_ln_vec<1>"),
    (256, False, "k_ln<8>"),
    (263, True, "k_ln<16>"),
    (384, True, "k_ln<16>"),
    (512, True, "k_ln_vec<2>"),
    (512, False, "k_ln<16>"),
    (768, True, "k_ln<32>"),
    (1024, True, "k_ln<32>"),
]
LN_KERNELS = sorted({k for _, _, k in LN_CASES})

# rows_to_split (stack.cu): eight columns per thread when d % 8 == 0 and the rows are 16-byte aligned, else one;
# the debug hook's `scalar` flag forces the second at any shape.
ROWS_TO_SPLIT = [
    # (kernel, hook arguments)
    ("k_rows_to_split8", dict(scalar=False)),
    ("k_rows_to_split", dict(scalar=True)),
]
