"""Builds tuning variants of libfbgpu.so (different eval-kernel launch shapes) for one-shot A/B runs on the GPU box."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from featurebase_b200 import build as B
VARIANTS = {   # name -> -D defines; edit freely, outputs featurebase_b200/libfbgpu_<name>.so (select with FBGPU_LIB=...)
    "gd_nopipe": ["FBGPU_GD_PIPE=0"],
    "pair_nopf": ["FBGPU_PAIR_NO_PF"],          # pair kernel without the L2 prefetch of the next unit's payload lines
    "pair_bm4": ["FBGPU_PAIR_BM_UNROLL=4"],     # pair kernel: bitmap x bitmap loop unrolled 4 (default 8)
    "addr_imad": ["FBGPU_ADDR_IMAD"],            # scatter / probe word addresses with IMAD.HI on the FMA pipe (measured slower: IMAD.HI is half rate)
    "wp_reg3": ["FBGPU_WP_REG_RING", "FBGPU_WP_RING=3"],   # word-parallel op loop with a REGISTER ring of 3 operand slices (22 us on config 3 in the round-2 first measurement)
    "wp_reg6": ["FBGPU_WP_REG_RING", "FBGPU_WP_RING=6"],   # register ring of 6 (30 us: the default of call 5)
    "wp_narrow": ["FBGPU_WP_NARROW"],                      # cp.async ring with 16 bytes per thread, 128 threads per CTA (19 us on config 3; default: 32 bytes, 64 threads)
    "wp_async4": ["FBGPU_WP_ASYNC_DEPTH=4"],               # cp.async shared-memory ring (default depth 8)
    "pair_w9": ["FBGPU_PAIR_WARPS=9"],                     # pair_count_kernel: 3 CTAs of 9 warps per SM (default 8)
    "pair_w7": ["FBGPU_PAIR_WARPS=7"],
    "pair_pf3": ["FBGPU_PAIR_PF_DIST=3"],                  # L2 prefetch three units ahead (default 1)
    "pair_w13b2": ["FBGPU_PAIR_WARPS=13", "FBGPU_PAIR_MIN_BLOCKS=2"],   # 2 CTAs of 13 warps
    "wp_legacy": ["FBGPU_WP_LEGACY_LOOP"],       # round-1 rotating-ring loop
    "pair_unscatter": ["FBGPU_PAIR_UNSCATTER"],
    "eval_deep1": ["FBGPU_EVAL_DEEP=1"],                                  # round-1 scatter loop: one chunk load in flight per lane
    "eval_mb8": ["FBGPU_EVAL_MIN_BLOCKS=8"],                              # round-1 shape: 32 registers, 8 CTAs / SM
    "eval_mb5": ["FBGPU_EVAL_MIN_BLOCKS=5"],                              # 48 registers, 5 CTAs / SM
    "eval_mb6_deep4": ["FBGPU_EVAL_MIN_BLOCKS=6", "FBGPU_EVAL_DEEP=4"],  # pair_count_kernel array x array: clear the a-side bits after the probe instead of wiping 8 KiB per pair
}
only = sys.argv[1:]
if only:
    VARIANTS = {k: v for k, v in VARIANTS.items() if k in only}
if __name__ == "__main__":
    for name, defs in VARIANTS.items():
        out = B.build_fbgpu(force=True, defines=defs, out_name=f"libfbgpu_{name}.so")
        print(out)
