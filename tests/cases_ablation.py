# coding=utf-8
"""Seeded rollout cases of the beam decoder without graph attention (use_gnn off, the reference scripts' default when
--use_gnn is not passed), shared by tests/golden/make_golden_ablation.py and the tests that read its goldens."""

# name: (oracle.default_config overrides, seed)
ROLLOUTS_NO_GNN = {
    # multifuture_inference.py's decode (K = 20 diverse, first step's scores zeroed) on the 36x18 grid: 60 beam rows
    # select the CTA-pair cell kernel
    "beam_k20_nognn": (dict(batch_size=3, use_grids=[True, False], use_beam_search=True, beam_size=20,
                            diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=False), 61),
    # test.py --use_beam_search: K = 5 plain beam on the 18x9 grid
    "beam_k5_nognn": (dict(batch_size=2, use_grids=[False, True], use_beam_search=True, beam_size=5,
                           diverse_beam=False, fix_num_timestep=0, use_gnn=False), 68),
}

# At size (the existing at-size rule of tests/test_parity_gpu.py): K = 20 diverse beam of 16 trajectories on 36x18, the
# shape of tests/golden/atsize_beam_k20_n16.npz without the attention; its golden holds reduced statistics
# (cases.rollout_stats) of the fp64 oracle, which the small cases above pin to the executed reference.
ROLLOUTS_NO_GNN_ATSIZE = {
    "beam_k20_nognn_n16": (dict(batch_size=16, use_grids=[True, False], use_beam_search=True, beam_size=20,
                                diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=False), 63),
}
