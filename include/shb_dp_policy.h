/*
 * shb_dp_policy.h — the ONE place where the tie-break rules of the overlap dynamic programme are chosen.
 *
 * In the reference the DP is seqan::globalAlignment (SeqAn 2.x, un-vendored, absent from the build container;
 * call sites src/AssemblerAlign3.cpp:117-122,254-260, src/Align4.cpp:1027-1033, src/AssemblerAlign1.cpp:129-135).
 * The SCORE of the result is that of any correct overlap alignment; WHICH of several co-optimal paths is
 * reported depends on three choices that no reference test pins (SURVEY.md F4, Appendix A: "UNVERIFIED"):
 *
 *   SHB_DP_DIAG_WINS_TIES    1: a diagonal move beats a gap move of equal score            (0: the gap move wins)
 *   SHB_DP_VERT_BEFORE_HORZ  1: of two gap moves of equal score the vertical one (consumes b,
 *                               read 1) wins                                               (0: the horizontal one)
 *   SHB_DP_END_FIRST_MAX     1: the end cell is the FIRST maximum met in column-major order over the cells of
 *                               the last row and of the last column                        (0: the LAST one)
 *
 * Defaults = the recollection of SeqAn 2.4 in SURVEY.md Appendix A (SingleTrace / GapsLeft: `_maxScore` keeps its left
 * argument on ties, called as (vertical, horizontal) then (diagonal, gap); DPScout replaces the best cell on strict >).
 *
 * This header is included by BOTH the CUDA kernels (shasta_b200/csrc/align_kernels.cuh) and the CPU oracle
 * (oracle/align_oracle.c), so a later check against real SeqAn touches this file only (build both with e.g.
 * -DSHB_DP_VERT_BEFORE_HORZ=0). That switch is tested: build() also compiles the library under each of the seven other
 * policies (`make -C shasta_b200/csrc policies`: shasta_b200/lib/dp_policy/libshasta_b200_policy<N>.so, N = the bits
 * below), and tests/test_gpu_dp_policies.py holds every policy's kernels to the oracle under the same policy. The oracle
 * can additionally switch policy at run time (orc_set_dp_policy) to measure how many candidate pairs are exposed to the
 * choice at all (bench.py: "policy_invariant_fraction").
 */
#ifndef SHB_DP_POLICY_H
#define SHB_DP_POLICY_H

#ifndef SHB_DP_DIAG_WINS_TIES
#define SHB_DP_DIAG_WINS_TIES 1
#endif
#ifndef SHB_DP_VERT_BEFORE_HORZ
#define SHB_DP_VERT_BEFORE_HORZ 1
#endif
#ifndef SHB_DP_END_FIRST_MAX
#define SHB_DP_END_FIRST_MAX 1
#endif

/* The three choices as one integer (bit 0, 1, 2 in the order above). */
#define SHB_DP_POLICY_BITS ((SHB_DP_DIAG_WINS_TIES ? 1 : 0) | (SHB_DP_VERT_BEFORE_HORZ ? 2 : 0) | (SHB_DP_END_FIRST_MAX ? 4 : 0))
#define SHB_DP_POLICY_COUNT 8

#endif
