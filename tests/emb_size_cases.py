# coding=utf-8
"""Configurations of the --emb_size goldens (tests/golden/make_golden_emb_size.py): oracle.multiverse_ref.default_config
overrides and seeds.  Every case has an x block wider than 64 channels in some cell."""

# name: (default_config overrides, seed)
ROLLOUTS = {
    # test.py --use_scene_enc --use_gnn --emb_size 128: greedy decode of both scales
    "greedy_two_scale_emb128": (dict(batch_size=3, emb_size=128, use_gnn=True), 91),
    # multifuture_inference.py --use_scene_enc --use_gnn --emb_size 128: K = 20 diverse beam on 36x18
    "beam_k20_emb128": (dict(batch_size=3, emb_size=128, use_grids=[True, False], use_beam_search=True, beam_size=20,
                             diverse_beam=True, diverse_gamma=0.01, fix_num_timestep=1, use_gnn=True), 92),
    # test.py --use_scene_enc --use_beam_search --emb_size 96 without --use_gnn: K = 5 plain beam on 18x9 (cpad 352)
    "beam_k5_emb96": (dict(batch_size=2, emb_size=96, use_grids=[False, True], use_beam_search=True, beam_size=5,
                           diverse_beam=False, fix_num_timestep=0, use_gnn=False), 93),
    # train.py's own model defaults: emb_size 128, no scene encoder, no attention, strides 2,4,8 on all three grids
    "defaults_three_grids": (dict(batch_size=2, emb_size=128, use_scene_enc=False, use_gnn=False,
                                  scene_grid_strides=[2, 4, 8], use_grids=[True, True, True]), 94),
}
# name: (overrides, seed) of one Model + Trainer step (loss weights 1.0 / 0.2, wd 0.001, Adadelta at 0.3, clip 10)
TRAIN = {
    "defaults_three_grids": (dict(ROLLOUTS["defaults_three_grids"][0]), 95),
    "scene_enc_emb96": (dict(batch_size=2, emb_size=96, use_gnn=True), 96),
}
TRAIN_ARGS = dict(grid_loss_weight=1.0, grid_reg_loss_weight=0.2, wd=0.001, init_lr=0.3, clip_gradient_norm=10.0,
                  optimizer="adadelta")
