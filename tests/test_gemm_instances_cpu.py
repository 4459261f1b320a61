"""The GPU tests' shape lists reach every wgmma GEMM instance and both sides of every split-K decision.

tests/gemm_instances.py restates the launchers' selection rules; this maps the shape lists of test_gemm_gpu.py and
test_gemm_a32_gpu.py through them.  Adding an instance or moving a threshold in csrc/ without a GPU case that runs it
fails here, without a GPU."""
import gemm_instances as gi
import test_gemm_a32_gpu as a32
import test_gemm_gpu as nt


def test_restated_rules_on_known_shapes():
    # the decoder's 2048-row linears: 16 x 4 tiles of 128 -> 64-wide tiles (gemm_a32_sm90.cu: `bn` in coda_gemm_a32)
    assert gi.gemm_a32(3, 2048, 512, 512, False)[0][1] == 64
    # one 128 x 64 tile over 530 slabs: 132 splits of 5, the last 26 empty
    assert gi.gemm_tn32(16960, 128, 64) == (64, 132, 26)
    # weight gradient over 200000 rows on 2 tiles: 132 splits asked; 3125 k-blocks at 24 per split fill 131 of them,
    # none is left empty
    inst, ksplit = gi.gemm_tn(3, 200000, 256, 128)
    assert inst == (3, 128, 2, False, True) and ksplit == 131
    assert gi.gemm_nt(1, True, 1, 256, 3072, 768) == ((1, 256, 4, True, False), 1)


def test_gemm_nt_cases_reach_every_instance_and_split():
    def pick(ns, f16, batch, m, n, k, bias, relu, ldc_pad):
        return gi.gemm_nt(ns, f16, batch, m, n, k, act=int(relu))

    picks = [(c, *pick(*c)) for c in nt.NT_CASES]
    assert {inst for _, inst, _ in picks} == gi.NT_INSTANCES
    splits = [c for c, _, ks in picks if ks > 1]
    assert splits and any(ks == 1 for _, _, ks in picks)
    # the split-K reduction applies the bias, walks the batch and writes rows ldc > n apart
    assert any(c[6] for c in splits) and any(c[2] > 1 for c in splits) and any(c[8] > 0 for c in splits)
    assert any(c[1] for c in splits)
    # a contraction long enough to split, but with ReLU: the fused epilogue runs instead
    assert any(c[7] and ks == 1 and gi.gemm_nt(c[0], c[1], c[2], c[3], c[4], c[5])[1] > 1 for c, _, ks in picks)
    for dim in (3, 4, 5):      # m, n, k at 1 and on either side of 64 and 128
        assert {1, 63, 64, 65, 127, 128, 129} <= {c[dim] for c in nt.NT_CASES}
    assert any(c[1] and c[4] <= 64 for c in nt.NT_CASES) and any(c[1] and c[4] == 512 for c in nt.NT_CASES)


def test_gemm_tn_cases_reach_every_instance_and_split():
    picks = [gi.gemm_tn(ns, mc, m, n) for ns, mc, m, n in nt.TN_CASES]
    assert {inst for inst, _ in picks} == gi.TN_INSTANCES
    assert {ks > 1 for _, ks in picks} == {False, True}
    assert {1, 65, 200000} <= {c[1] for c in nt.TN_CASES}
    # the 2- and 3-wide heads' weight gradients, on two planes, with and without split-K
    heads = [(c, ks) for c, (_, ks) in zip(nt.TN_CASES, picks) if c[0] == 2 and min(c[2], c[3]) in (2, 3)]
    assert {min(c[2], c[3]) for c, _ in heads} == {2, 3} and {ks > 1 for _, ks in heads} == {False, True}


def test_gemm_a32_cases_reach_every_instance_and_grid():
    def pick(ns, m, n, k, b_mn, mode, stats, relu):
        return gi.gemm_a32(ns, m, n, k, b_mn, mode, stats)

    picks = [(c, *pick(*c)) for c in a32.A32_CASES]
    assert {inst for _, inst, _ in picks} == gi.A32_INSTANCES
    assert {res for _, _, res in picks} == {False, True}
    assert any(res and c[6] for c, _, res in picks)                 # B-resident grid with column statistics
    assert any(c[6] and c[1] % 128 for c, _, _ in picks)            # statistics with a ragged last tile
    # both sides of the 64 / 128 tile-width switch at the same n
    widths = {}
    for c, inst, _ in picks:
        widths.setdefault(c[2], set()).add(inst[1])
    assert any(w == {64, 128} for w in widths.values())
    assert {12, 200, 4096} <= {c[3] for c in a32.A32_CASES if c[4]}     # b_mn contraction lengths
    assert {1, 64, 127} <= {c[1] for c in a32.A32_CASES}
    # prologues whose per-k vectors are padded past k
    assert {a32.AFFINE_RELU, a32.BN_BWD} <= {c[5] for c in a32.A32_CASES if c[3] % 64}


def test_gemm_tn32_cases_reach_every_width_and_split():
    picks = [(c, *gi.gemm_tn32(c[0], c[1], c[2])) for c in a32.TN32_CASES]
    assert {bn for _, bn, _, _ in picks} == gi.TN32_INSTANCES
    assert {ks > 1 for _, _, ks, _ in picks} == {False, True}
    assert any(empty > 0 for _, _, _, empty in picks)
    # no split with >= 132 output tiles: the column sums are stored by the GEMM itself
    assert any(ks == 1 and -(-c[1] // 128) * -(-c[2] // bn) >= gi.SMS for c, bn, ks, _ in picks)
    # the tail slab in the two-input BatchNorm-backward mode, on either side of the split
    tails = [(c, ks) for c, _, ks, _ in picks if c[3] == a32.BN_BWD and c[0] % 32]
    assert {1, 31, 33} <= {c[0] for c, _ in tails} and {ks > 1 for _, ks in tails} == {False, True}
    assert {1, 31, 33} <= {c[0] for c in a32.TN32_CASES if c[3] == a32.PLAIN}
    assert any(c[3] == a32.PLAIN and c[0] % 32 and ks > 1 for c, _, ks, _ in picks)
    assert any(c[5] for c in a32.TN32_CASES)                       # column slices of wider matrices
    assert {c[6] for c in a32.TN32_CASES if c[3] in (a32.POOLED, a32.POOLED_PRE)} == {32, 128, 256}
