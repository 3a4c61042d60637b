"""CPU-side build evidence (cuobjdump on the in-tree libdfgpu.so) for Right joins in the fused pipeline (DFGPU_STAGE_RIGHT): the seven
instantiations that run them exist and fit the registers their launch bounds allow, and every other function of the library is the one
the build before them had.  The RIGHT path lives only in new instantiations (pipe_kernel VAR bit 1024, pipe_output_right_kernel); the
interpreters' nullable-payload parameter defaults to the old behaviour, so PARENT lists, per function of that build, its registers, stack
and local memory and a hash of its SASS instructions, and none of them may move."""
import hashlib
import re
import subprocess

import pytest

from datafusion_b200 import capi

PK = "_ZN5dfgpu11pipe_kernelILi{}ELb{}ELi{}EEEvPKNS_10PipeParamsElPy"
# function: the registers its launch bounds allow (256 threads; 3 blocks per SM for the unordered output and hash sinks, 2 for the dense one)
NEW = {
    PK.format(5, 0, 2 | 512 | 1024): 80, PK.format(5, 1, 512 | 1024): 80,      # unordered output (with bitmaps), integer and Decimal128
    PK.format(7, 0, 1024): 128, PK.format(7, 1, 1024): 128,                    # dense aggregate sink
    PK.format(8, 0, 1024): 80, PK.format(8, 1, 1024): 80,                      # hash aggregate sink
    "_ZN5dfgpu24pipe_output_right_kernelEPKNS_10PipeParamsElNS_7OutColsEPyPjS4_S4_": 255,   # ordered output
}
# function: (REG, STACK, LOCAL, first 16 hex digits of the SHA-1 of its SASS instructions, one per line without addresses or encodings)
PARENT = {
    "_ZN5dfgpu11iota_kernelEPjl": (28, 0, 0, "5b19e902d997b53b"),
    "_ZN5dfgpu11pipe_kernelILi2ELb0ELi0EEEvPKNS_10PipeParamsElPy": (80, 304, 0, "da32bb86053d1160"),
    "_ZN5dfgpu11pipe_kernelILi2ELb0ELi256EEEvPKNS_10PipeParamsElPy": (80, 496, 0, "a659395abfe0711c"),
    "_ZN5dfgpu11pipe_kernelILi2ELb1ELi0EEEvPKNS_10PipeParamsElPy": (80, 608, 0, "adb57ce5b8bfa0ed"),
    "_ZN5dfgpu11pipe_kernelILi2ELb1ELi256EEEvPKNS_10PipeParamsElPy": (80, 768, 0, "fc32237a568309c8"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi0EEEvPKNS_10PipeParamsElPy": (80, 384, 0, "e022b975ed7abcbd"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi11EEEvPKNS_10PipeParamsElPy": (80, 432, 0, "eebc9245288661c8"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi192EEEvPKNS_10PipeParamsElPy": (80, 56, 0, "0e14056ef1dbbbcf"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi1EEEvPKNS_10PipeParamsElPy": (80, 384, 0, "c83176520e64d7eb"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi267EEEvPKNS_10PipeParamsElPy": (80, 544, 0, "d4be8b12daecbac2"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi2EEEvPKNS_10PipeParamsElPy": (80, 384, 0, "a86c2274a98961e7"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi3EEEvPKNS_10PipeParamsElPy": (80, 384, 0, "836b5f5174d39570"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi43EEEvPKNS_10PipeParamsElPy": (80, 416, 0, "b3a304563f516c3a"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi72EEEvPKNS_10PipeParamsElPy": (80, 112, 0, "07f50672be231c04"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi8EEEvPKNS_10PipeParamsElPy": (80, 432, 0, "2a3ba39d8f7bf7ba"),
    "_ZN5dfgpu11pipe_kernelILi3ELb0ELi9EEEvPKNS_10PipeParamsElPy": (80, 432, 0, "ab0c6adee3420424"),
    "_ZN5dfgpu11pipe_kernelILi3ELb1ELi0EEEvPKNS_10PipeParamsElPy": (80, 704, 0, "c88e6b0285d4ea7a"),
    "_ZN5dfgpu11pipe_kernelILi3ELb1ELi256EEEvPKNS_10PipeParamsElPy": (80, 800, 0, "686669423e5e74d9"),
    "_ZN5dfgpu11pipe_kernelILi5ELb0ELi0EEEvPKNS_10PipeParamsElPy": (80, 288, 0, "aa534d62a74d0ba9"),
    "_ZN5dfgpu11pipe_kernelILi5ELb0ELi258EEEvPKNS_10PipeParamsElPy": (80, 464, 0, "a008cf7bc90a657a"),
    "_ZN5dfgpu11pipe_kernelILi5ELb0ELi2EEEvPKNS_10PipeParamsElPy": (80, 288, 0, "f303f4b0a51f1a4a"),
    "_ZN5dfgpu11pipe_kernelILi5ELb0ELi514EEEvPKNS_10PipeParamsElPy": (80, 304, 0, "1e3b9e0839ad6560"),
    "_ZN5dfgpu11pipe_kernelILi5ELb0ELi770EEEvPKNS_10PipeParamsElPy": (80, 464, 0, "3bae729457b18b8f"),
    "_ZN5dfgpu11pipe_kernelILi5ELb1ELi0EEEvPKNS_10PipeParamsElPy": (80, 592, 0, "ca58f28c2f677f08"),
    "_ZN5dfgpu11pipe_kernelILi5ELb1ELi256EEEvPKNS_10PipeParamsElPy": (80, 752, 0, "62cacf20d84d26a5"),
    "_ZN5dfgpu11pipe_kernelILi5ELb1ELi512EEEvPKNS_10PipeParamsElPy": (80, 592, 0, "cb128853a8211219"),
    "_ZN5dfgpu11pipe_kernelILi5ELb1ELi768EEEvPKNS_10PipeParamsElPy": (80, 768, 0, "33791312bd3a5550"),
    "_ZN5dfgpu11pipe_kernelILi6ELb0ELi0EEEvPKNS_10PipeParamsElPy": (80, 304, 0, "1eac37b6f4d32886"),
    "_ZN5dfgpu11pipe_kernelILi6ELb0ELi258EEEvPKNS_10PipeParamsElPy": (80, 496, 0, "5086b40340810491"),
    "_ZN5dfgpu11pipe_kernelILi6ELb0ELi2EEEvPKNS_10PipeParamsElPy": (80, 304, 0, "99da24fb24868d36"),
    "_ZN5dfgpu11pipe_kernelILi6ELb0ELi34EEEvPKNS_10PipeParamsElPy": (80, 336, 0, "ae9dc82c2b670e52"),
    "_ZN5dfgpu11pipe_kernelILi6ELb0ELi64EEEvPKNS_10PipeParamsElPy": (128, 24, 0, "862e07740cfabc68"),
    "_ZN5dfgpu11pipe_kernelILi6ELb1ELi0EEEvPKNS_10PipeParamsElPy": (80, 608, 0, "8c29df627661978e"),
    "_ZN5dfgpu11pipe_kernelILi6ELb1ELi256EEEvPKNS_10PipeParamsElPy": (80, 784, 0, "7b61fc4239cb5b1e"),
    "_ZN5dfgpu11pipe_kernelILi7ELb0ELi0EEEvPKNS_10PipeParamsElPy": (128, 336, 0, "d2f494814cb059e9"),
    "_ZN5dfgpu11pipe_kernelILi7ELb0ELi256EEEvPKNS_10PipeParamsElPy": (128, 432, 0, "1aff5d7b6759f9b8"),
    "_ZN5dfgpu11pipe_kernelILi7ELb1ELi0EEEvPKNS_10PipeParamsElPy": (128, 608, 0, "1d3793caacdb8d2f"),
    "_ZN5dfgpu11pipe_kernelILi7ELb1ELi256EEEvPKNS_10PipeParamsElPy": (128, 720, 0, "2c86d7867be9a129"),
    "_ZN5dfgpu11pipe_kernelILi8ELb0ELi0EEEvPKNS_10PipeParamsElPy": (80, 400, 0, "7828a7feb8e1599a"),
    "_ZN5dfgpu11pipe_kernelILi8ELb0ELi256EEEvPKNS_10PipeParamsElPy": (80, 496, 0, "5e7da7608e81cb4f"),
    "_ZN5dfgpu11pipe_kernelILi8ELb1ELi0EEEvPKNS_10PipeParamsElPy": (80, 720, 0, "c15008297b3903cb"),
    "_ZN5dfgpu11pipe_kernelILi8ELb1ELi256EEEvPKNS_10PipeParamsElPy": (80, 800, 0, "7de894d163b1120e"),
    "_ZN5dfgpu11salt_kernelEPtl": (30, 0, 0, "940cbb6854416ed0"),
    "_ZN5dfgpu11take_kernelINS_3B16EEEvPKT_PKhlPKjlPS2_Pj": (31, 0, 0, "ee533c13fd52bb59"),
    "_ZN5dfgpu11take_kernelIhEEvPKT_PKhlPKjlPS1_Pj": (26, 0, 0, "29940f1f1da79102"),
    "_ZN5dfgpu11take_kernelIjEEvPKT_PKhlPKjlPS1_Pj": (30, 0, 0, "c36d02f11a8987d4"),
    "_ZN5dfgpu11take_kernelImEEvPKT_PKhlPKjlPS1_Pj": (30, 0, 0, "a759bd3d181d1772"),
    "_ZN5dfgpu11take_kernelItEEvPKT_PKhlPKjlPS1_Pj": (30, 0, 0, "9efaab1bfea85261"),
    "_ZN5dfgpu14col_sum_kernelENS_6ColRefElPy": (32, 0, 0, "01284739f509feca"),
    "_ZN5dfgpu15agg_emit_kernelENS_8EmitDescEPKjlPvPjS4_": (32, 0, 0, "72ab8fa799959f91"),
    "_ZN5dfgpu15fill_u64_kernelEPymy": (12, 0, 0, "141f269f9f75dc3b"),
    "_ZN5dfgpu15l2_flush_kernelEP4int4m": (14, 0, 0, "4e80ae00df8fd95d"),
    "_ZN5dfgpu15wide_key_kernelENS_11WideKeyColsEliPyPj": (29, 0, 0, "95306822054b6899"),
    "_ZN5dfgpu16expr_eval_kernelENS_8EProgramElPvPjS2_S2_Pi": (32, 160, 0, "04413d102b8aa37a"),
    "_ZN5dfgpu16fill_pair_kernelEP10ulonglong2mS0_": (14, 0, 0, "eedf70a882157331"),
    "_ZN5dfgpu16hash_init_kernelEPymiNS_9HashIdentE": (32, 128, 0, "76874a0be4dd0dc3"),
    "_ZN5dfgpu16join_emit_kernelILb0EEEvlPKjS2_S2_PKmiPjS5_": (32, 0, 0, "e7e8c6a62a00a7c7"),
    "_ZN5dfgpu16join_emit_kernelILb1EEEvlPKjS2_S2_PKmiPjS5_": (32, 0, 0, "678dce20fb74bd9a"),
    "_ZN5dfgpu16mark_bits_kernelEPKjlPj": (16, 0, 0, "575d33ea83e2e7a9"),
    "_ZN5dfgpu16pack_keys_kernelENS_14PackKeysParamsEl": (76, 0, 0, "ac7c48d23c7ce003"),
    "_ZN5dfgpu16take_bool_kernelEPKhlS1_lPKjlPjS4_": (18, 0, 0, "aa76d50a3f858fd8"),
    "_ZN5dfgpu17agg_rehash_kernelILi1EEEvNS_8TableDevES1_NS_9AccArraysE": (24, 0, 0, "f3d764fb50a9bf0d"),
    "_ZN5dfgpu17agg_rehash_kernelILi2EEEvNS_8TableDevES1_NS_9AccArraysE": (26, 0, 0, "9efb3106e8bca3ce"),
    "_ZN5dfgpu17agg_update_kernelILi1ELi4ELb0EEEvNS_9GroupColsENS_6AggSetENS_8TableDevEllPKjPjPy": (48, 24, 0, "6bfcb503596255b9"),
    "_ZN5dfgpu17agg_update_kernelILi1ELi4ELb1EEEvNS_9GroupColsENS_6AggSetENS_8TableDevEllPKjPjPy": (58, 0, 0, "11e6d242fbc4216d"),
    "_ZN5dfgpu17agg_update_kernelILi2ELi4ELb0EEEvNS_9GroupColsENS_6AggSetENS_8TableDevEllPKjPjPy": (70, 0, 0, "4640ee859986dcbb"),
    "_ZN5dfgpu17agg_update_kernelILi2ELi4ELb1EEEvNS_9GroupColsENS_6AggSetENS_8TableDevEllPKjPjPy": (64, 64, 0, "8659e2f24c3c59c1"),
    "_ZN5dfgpu17bloom_fold_kernelEPK10ulonglong2Pym": (14, 0, 0, "47e8cfc18c5cd4ce"),
    "_ZN5dfgpu17col_minmax_kernelENS_6ColRefEliPy": (32, 0, 0, "2dae292752bb6184"),
    "_ZN5dfgpu17dict_remap_kernelIaEEvPKT_PKhllPKilPiPjS8_": (20, 0, 0, "c96ab22b108c70c6"),
    "_ZN5dfgpu17dict_remap_kernelIhEEvPKT_PKhllPKilPiPjS8_": (19, 0, 0, "d26e465008df9758"),
    "_ZN5dfgpu17dict_remap_kernelIiEEvPKT_PKhllPKilPiPjS8_": (18, 0, 0, "3af14473f61e1731"),
    "_ZN5dfgpu17dict_remap_kernelIjEEvPKT_PKhllPKilPiPjS8_": (18, 0, 0, "07af034e3c63087d"),
    "_ZN5dfgpu17dict_remap_kernelIlEEvPKT_PKhllPKilPiPjS8_": (19, 0, 0, "7787b027a6d25b65"),
    "_ZN5dfgpu17dict_remap_kernelIsEEvPKT_PKhllPKilPiPjS8_": (20, 0, 0, "73e2fbf3c54382f6"),
    "_ZN5dfgpu17dict_remap_kernelItEEvPKT_PKhllPKilPiPjS8_": (19, 0, 0, "ad004d65419f9eb0"),
    "_ZN5dfgpu17flags_emit_kernelEPKjliPKmPj": (22, 0, 0, "c41fa6fcca989e41"),
    "_ZN5dfgpu17join_build_kernelENS_7KeyColsElNS_8TableRefEPy": (29, 0, 0, "8a00646a185635e6"),
    "_ZN5dfgpu17radix_hist_kernelEPKyliPy": (26, 0, 0, "5b1418587f87c2ce"),
    "_ZN5dfgpu17scan_tiles_kernelILi1024EEEvPmlS1_": (48, 0, 0, "95104e5a825bdda9"),
    "_ZN5dfgpu18flags_count_kernelEPKjliPm": (28, 0, 0, "ba9546251afe3571"),
    "_ZN5dfgpu18hash_rehash_kernelEPKymPymi": (32, 0, 0, "c5989bfc6e56037a"),
    "_ZN5dfgpu18join_minmax_kernelENS_7KeyColsEliPy": (48, 0, 0, "b827f387eb842c35"),
    "_ZN5dfgpu18lookup_emit_kernelENS_9LookupDevEPKjliNS_8EmitColsE": (40, 0, 0, "57474713261755ab"),
    "_ZN5dfgpu18lookup_init_kernelEPymi": (20, 0, 0, "6f9338d6756f9a42"),
    "_ZN5dfgpu18pipe_output_kernelILb0EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_": (80, 592, 0, "6f73ad9369eccad9"),
    "_ZN5dfgpu18pipe_output_kernelILb1EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_": (80, 800, 0, "71995c530ba08957"),
    "_ZN5dfgpu18radix_probe_kernelILi1ELb0EEEvPKNS_8RadixRecElNS_9InlineRefENS_8RadixOutEPjPy": (45, 128, 0, "b4b04137b96b35b8"),
    "_ZN5dfgpu18radix_probe_kernelILi1ELb1EEEvPKNS_8RadixRecElNS_9InlineRefENS_8RadixOutEPjPy": (48, 0, 0, "67117a1e42ef9dfc"),
    "_ZN5dfgpu18radix_probe_kernelILi2ELb0EEEvPKNS_8RadixRecElNS_9InlineRefENS_8RadixOutEPjPy": (56, 128, 0, "1d6490cae9319667"),
    "_ZN5dfgpu18radix_probe_kernelILi2ELb1EEEvPKNS_8RadixRecElNS_9InlineRefENS_8RadixOutEPjPy": (62, 0, 0, "d37f8459f9df9b29"),
    "_ZN5dfgpu18scatter_u32_kernelEPKjlPj": (32, 0, 0, "f4d71490279d6d39"),
    "_ZN5dfgpu19filter_fused_kernelILi0EEEvPKNS_8EProgramEPKlillNS_10FilterColsEPyPjS7_Pi": (40, 160, 0, "44650b62d7243237"),
    "_ZN5dfgpu19filter_fused_kernelILi1EEEvPKNS_8EProgramEPKlillNS_10FilterColsEPyPjS7_Pi": (32, 0, 0, "5a36227c62a215d6"),
    "_ZN5dfgpu19filter_fused_kernelILi2EEEvPKNS_8EProgramEPKlillNS_10FilterColsEPyPjS7_Pi": (62, 288, 0, "4db85d423fb56199"),
    "_ZN5dfgpu19generate_i64_kernelEimllllPl": (30, 0, 0, "afbff696b2981458"),
    "_ZN5dfgpu19radix_prefix_kernelEPKyiPyS2_": (32, 0, 0, "0cc226daef3168e6"),
    "_ZN5dfgpu20agg_init_seen_kernelILi1EEEvNS_8TableDevEPh": (16, 0, 0, "3870aae0e8289715"),
    "_ZN5dfgpu20agg_init_seen_kernelILi2EEEvNS_8TableDevEPh": (16, 0, 0, "2a1e1b6b8e53a711"),
    "_ZN5dfgpu20agg_occupancy_kernelILi1EEEvNS_8TableDevEPj": (16, 0, 0, "49f79c8f2d81b3bd"),
    "_ZN5dfgpu20agg_occupancy_kernelILi2EEEvNS_8TableDevEPj": (16, 0, 0, "45a1beff2e97fa0d"),
    "_ZN5dfgpu20expr_eval_dec_kernelENS_8EProgramElPvPjS2_S2_Pi": (48, 272, 0, "e225811fc0e976d1"),
    "_ZN5dfgpu20lookup_groups_kernelENS_9LookupDevEiiPj": (18, 0, 0, "a19c63b2a7190222"),
    "_ZN5dfgpu20lookup_rehash_kernelENS_9LookupDevES0_": (32, 0, 0, "dc344c644bf46514"),
    "_ZN5dfgpu20mark_from_idx_kernelEPKjlPj": (16, 0, 0, "fc6d1cb67f4e41ab"),
    "_ZN5dfgpu21agg_fold_pairs_kernelEP10ulonglong2PyS2_m": (20, 0, 0, "aadee07a08545255"),
    "_ZN5dfgpu21bitmap_or_copy_kernelEPjlPKhll": (30, 0, 0, "2bb725659534d5ba"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi1EEEvPKlllPj": (40, 0, 0, "7d98637361148e97"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi2EEEvPKlllPj": (40, 0, 0, "78ad5672072f0991"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi3EEEvPKlllPj": (40, 0, 0, "bb3464c19d34c065"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi4EEEvPKlllPj": (40, 0, 0, "cff59febb93229dd"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi5EEEvPKlllPj": (40, 0, 0, "2fd7db26ee7a825f"),
    "_ZN5dfgpu21cmp_i64_scalar_kernelILi6EEEvPKlllPj": (40, 0, 0, "5586f4b65c1e9756"),
    "_ZN5dfgpu21mark_null_keys_kernelEPKhllPj": (47, 0, 0, "cafbb5387ae17960"),
    "_ZN5dfgpu21partition_hist_kernelENS_8PartKeysElilPy": (28, 0, 0, "a88c9f68810206f5"),
    "_ZN5dfgpu21pipe_probe_agg_kernelEPK10ulonglong2lNS_9LookupDevEiiPjPy": (47, 0, 0, "24964997d066718e"),
    "_ZN5dfgpu22agg_update_fast_kernelILi2ELi1ELi1EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (46, 0, 0, "731400c4875f85fb"),
    "_ZN5dfgpu22agg_update_fast_kernelILi2ELi2ELi1EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (46, 0, 0, "7c599535afd88e32"),
    "_ZN5dfgpu22agg_update_fast_kernelILi2ELi3ELi1EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (48, 16, 0, "dd5b1521f177d649"),
    "_ZN5dfgpu22agg_update_fast_kernelILi2ELi4ELi1EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (56, 0, 0, "db012a3238e8340c"),
    "_ZN5dfgpu22agg_update_fast_kernelILi4ELi1ELi0EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (48, 16, 0, "809285c8b8adc0cc"),
    "_ZN5dfgpu22agg_update_fast_kernelILi4ELi2ELi0EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (62, 0, 0, "e1aa1da87706aa12"),
    "_ZN5dfgpu22agg_update_fast_kernelILi4ELi2ELi1EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (80, 8, 0, "37802d4764825dd3"),
    "_ZN5dfgpu22agg_update_fast_kernelILi4ELi3ELi0EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (64, 16, 0, "c1bcb332051c4aed"),
    "_ZN5dfgpu22agg_update_fast_kernelILi4ELi4ELi0EEEvPKyNS_8FastAggsENS_8TableDevEllPKjPjPy": (64, 40, 0, "42c98dbdd2cf3b2a"),
    "_ZN5dfgpu22agg_update_pair_kernelILi2ELb0EEEvPKyS2_S2_P10ulonglong2NS_8TableDevEllPKjPjPy": (48, 0, 0, "5603e0426836088e"),
    "_ZN5dfgpu22agg_update_pair_kernelILi2ELb1EEEvPKyS2_S2_P10ulonglong2NS_8TableDevEllPKjPjPy": (48, 0, 0, "5603e0426836088e"),
    "_ZN5dfgpu22agg_update_pair_kernelILi3ELb1EEEvPKyS2_S2_P10ulonglong2NS_8TableDevEllPKjPjPy": (64, 0, 0, "c11fbdb243bc9eff"),
    "_ZN5dfgpu22agg_update_pair_kernelILi4ELb0EEEvPKyS2_S2_P10ulonglong2NS_8TableDevEllPKjPjPy": (80, 0, 0, "b55eef2bb885d1ef"),
    "_ZN5dfgpu22agg_verify_wide_kernelENS_9GroupColsENS_8TableDevEllPi": (28, 0, 0, "3fdad7a9dc265832"),
    "_ZN5dfgpu22bitmap_popcount_kernelEPKhllPy": (30, 0, 0, "df17e5cdd69d5ba4"),
    "_ZN5dfgpu22lookup_init_acc_kernelENS_9LookupDevEiy": (16, 0, 0, "2f83ee6c6ca8540c"),
    "_ZN5dfgpu22partition_flags_kernelENS_8PartKeysEliPj": (28, 0, 0, "77951cafe11bdef8"),
    "_ZN5dfgpu22partition_hist8_kernelILb0EEEvNS_8PartKeysElilPy": (30, 0, 0, "138cdd3ee948abb5"),
    "_ZN5dfgpu22partition_hist8_kernelILb1EEEvNS_8PartKeysElilPy": (24, 0, 0, "85f7a8c9f6eccd37"),
    "_ZN5dfgpu23bitmap_set_range_kernelEPjll": (19, 0, 0, "faaf02f943ed08f7"),
    "_ZN5dfgpu23join_bloom_build_kernelENS_7KeyColsElPym": (27, 0, 0, "40db58f3b59496e5"),
    "_ZN5dfgpu23join_build_flags_kernelENS_7KeyColsElNS_8TableRefEPj": (32, 0, 0, "231123a56b39924f"),
    "_ZN5dfgpu23join_probe_count_kernelILb0EEEvNS_7KeyColsElNS_8TableRefEiiPjS3_PmPy": (26, 0, 0, "887ad1cacd4d9653"),
    "_ZN5dfgpu23join_probe_count_kernelILb1EEEvNS_7KeyColsElNS_8TableRefEiiPjS3_PmPy": (23, 0, 0, "12930eeff976051e"),
    "_ZN5dfgpu23join_probe_fused_kernelENS_7KeyColsElNS_8TableRefEiNS_9FusedColsEPyPjS3_": (32, 0, 0, "e96dc85615f24bd8"),
    "_ZN5dfgpu23lookup_scan_emit_kernelENS_9LookupDevEiNS_8EmitColsEPjPyS3_m": (32, 0, 0, "1785c83b00f3406f"),
    "_ZN5dfgpu23pipe_output_cols_kernelILb0EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_": (80, 592, 0, "964a29e19d310197"),
    "_ZN5dfgpu23pipe_output_cols_kernelILb1EEEvPKNS_10PipeParamsElNS_7OutColsEPyPjS5_S5_": (80, 816, 0, "3facab7d582fd208"),
    "_ZN5dfgpu24agg_convert_state_kernelENS_6AggSetENS_9StateOutsEl": (32, 0, 0, "6be3f96659286047"),
    "_ZN5dfgpu24join_build_inline_kernelILi1EEEvNS_7KeyColsENS_11PayloadColsElNS_9InlineRefEPy": (26, 0, 0, "48fe631cedfd9d97"),
    "_ZN5dfgpu24join_build_inline_kernelILi2EEEvNS_7KeyColsENS_11PayloadColsElNS_9InlineRefEPy": (32, 0, 0, "c9daa885a1afd515"),
    "_ZN5dfgpu24join_probe_inline_kernelILi1ELb0EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (32, 0, 0, "12d0e93446898a6e"),
    "_ZN5dfgpu24join_probe_inline_kernelILi1ELb1EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (38, 0, 0, "bdb429b076aa3fa8"),
    "_ZN5dfgpu24join_probe_inline_kernelILi2ELb0EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (43, 0, 0, "697c81a4b6a94c95"),
    "_ZN5dfgpu24join_probe_inline_kernelILi2ELb1EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (43, 0, 0, "fa26ba6a0b29415c"),
    "_ZN5dfgpu24partition_scatter_kernelILb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEl": (64, 0, 0, "a4e9494edc92266f"),
    "_ZN5dfgpu24partition_scatter_kernelILb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEl": (61, 0, 0, "eedd5d2c788515ae"),
    "_ZN5dfgpu24radix_scatter_tma_kernelEPKyS1_liPyPNS_8RadixRecE": (80, 32, 0, "c9bfeebfbf395be6"),
    "_ZN5dfgpu25lookup_insert_part_kernelENS_9LookupDevEPK10ulonglong2liPjPy": (34, 0, 0, "dede7369d08edfac"),
    "_ZN5dfgpu25partition_scatter8_kernelILb0ELb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli": (64, 0, 0, "cd03afec7c5ea306"),
    "_ZN5dfgpu25partition_scatter8_kernelILb0ELb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli": (64, 0, 0, "275f8de95af9c509"),
    "_ZN5dfgpu25partition_scatter8_kernelILb1ELb0EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli": (64, 0, 0, "b99f81d6edd89034"),
    "_ZN5dfgpu25partition_scatter8_kernelILb1ELb1EEEvNS_8PartKeysENS_8PartColsENS_8PartBitsElilPKyNS_7PeerDstEli": (64, 0, 0, "f8208785b0065a57"),
    "_ZN5dfgpu25radix_hist_records_kernelEPKyliPy": (26, 0, 0, "ee701e8fe75c5b64"),
    "_ZN5dfgpu28filter_allreduce_peer_kernelENS_9PeerWordsEiim": (34, 0, 0, "c3932a7c7d94408f"),
    "_ZN5dfgpu28lookup_filter_records_kernelENS_9LookupDevEPK10ulonglong2l": (24, 0, 0, "f8c0ff8cab026b37"),
    "_ZN5dfgpu28lookup_insert_records_kernelENS_9LookupDevEPK10ulonglong2liPy": (26, 0, 0, "c3923298bb7b1e43"),
    "_ZN5dfgpu28radix_scatter_records_kernelEPKyliPyPNS_8RadixRecE": (62, 32, 0, "0615025ba6bd82cb"),
    "_ZN5dfgpu31join_probe_inline_staged_kernelILi1EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (40, 0, 0, "6739e9b51edd2576"),
    "_ZN5dfgpu31join_probe_inline_staged_kernelILi2EEEvNS_7KeyColsElNS_9InlineRefENS_9InlineOutEPyPjS4_": (46, 0, 0, "e8a1404ab8a9425f"),
}


@pytest.fixture(scope="module")
def listing():
    use = subprocess.run(["cuobjdump", "-res-usage", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    res = {m.group(1): dict(kv.split(":") for kv in m.group(2).split()) for m in re.finditer(r"Function (\S+):\s*\n\s*(REG:.*)", use)}
    out = subprocess.run(["cuobjdump", "-sass", capi.LIB_PATH], capture_output=True, text=True, check=True).stdout
    code, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s+Function : (\S+)", line)
        if m:
            fn = m.group(1)
            code[fn] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,5}\*/\s+(.*?)\s*/\*", line)
        if fn and m:
            code[fn].append(m.group(1))
    return res, code


@pytest.mark.parametrize("fn", sorted(NEW))
def test_right_join_instantiations_exist_and_fit_their_launch_bounds(listing, fn):
    res, code = listing
    assert fn in res and fn in code, fn
    assert int(res[fn]["REG"]) <= NEW[fn], res[fn]


def test_the_library_has_no_other_new_function(listing):
    res, _ = listing
    assert sorted(set(res) - set(PARENT)) == sorted(NEW)


@pytest.mark.parametrize("fn", sorted(PARENT))
def test_existing_kernels_are_unchanged(listing, fn):
    res, code = listing
    assert fn in res and fn in code, fn
    got = (int(res[fn]["REG"]), int(res[fn]["STACK"]), int(res[fn]["LOCAL"]), hashlib.sha1("\n".join(code[fn]).encode()).hexdigest()[:16])
    assert got == PARENT[fn], (fn, got)
