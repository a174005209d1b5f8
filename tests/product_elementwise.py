"""The launches of twg_elementwise.cu's entry points in the product's training step, the cases beside them, and the
host-side launch geometry of the reductions among them (so that the CPU calibration in test_cpu_reduction_error_model.py
and the GPU suite in test_gpu_elementwise_conformance.py read one literal and one copy of each grid rule)."""

# Harvested by test_gpu_elementwise_conformance.elementwise_keys over tests/product_launches.py.  A change that adds,
# removes or re-dispatches one of these launches must update this set; each key is a case of the stage test.  Float
# fields are the fp32 value the kernel receives, to 6 significant digits.  Key layouts:
#   twg_bias_lrelu_fwd: rows, C, lrelu_on, non-null optional pointers (bias, planes, mask)
#   twg_lrelu_bwd: n
#   twg_lrelu_bwd_colsum: rows, C, lrelu_on, poolH, poolW, accumulate, non-null optional pointers (ref, mask, out, planes)
#   twg_colsum: rows, C, accumulate
#   twg_pool2: N, H, W, C, scale, outputs (out, planes)
#   twg_upsample2: N, H, W, C, scale
#   twg_upsample_concat: N, H, W, Ca, Cb, Nb, outputs (out, planes)
#   twg_upsample_concat_bwd: N, H, W, Ca, Cb, Nb
#   twg_axpby: n, 'y' when y was passed, alpha, beta
#   twg_scale_by_dev: n, alpha
#   twg_copy_cols: rows, Csrc, src_off, Cdst, dst_off, ncols
#   twg_mbstd_fwd: N, P, C, Ct, groups, 's_out' when passed;  twg_mbstd_bwd / _bwd2: N, P, C, Ct, groups
#   twg_sigmoid_ce: n, label, accumulate, 'grad' when passed
#   twg_logit_mean / _bwd: n, sign, margin, kind
#   twg_l1: n, accumulate, 'grad' when passed
#   twg_dragan_xhat: N, per_sample
#   twg_grad_penalty: N, per_sample, accumulate
#   twg_scale_rows: N, per_sample, 'scalar' when the device scalar was passed
#   twg_fanout_fwd: B, per_sample;  twg_fanout_bwd: B, per_sample, non-null optional pointers
#   twg_l1_groups: groups, per_group
#   twg_scale_groups2: per_group, sign, non-null gl0 / gl1
#   twg_gan_losses: B;  twg_gan_losses_bwd: B, non-null g0 .. g5
#   twg_sum_scalars: n, scale
#   twg_adam / twg_adam_dev_lr: n, beta1, beta2, eps
PRODUCT_ELEMENTWISE = {
    'twg_adam_dev_lr': [   (1184272, 0.5, 0.99, 1e-08), (1185296, 0.5, 0.99, 1e-08), (3285000, 0.5, 0.99, 1e-08),
                           (3287048, 0.5, 0.99, 1e-08), (4137488, 0.5, 0.99, 1e-08), (4140064, 0.5, 0.99, 1e-08),
                           (4269840, 0.5, 0.99, 1e-08), (4273440, 0.5, 0.99, 1e-08), (5645320, 0.5, 0.99, 1e-08),
                           (5647368, 0.5, 0.99, 1e-08), (5651464, 0.5, 0.99, 1e-08), (7090704, 0.5, 0.99, 1e-08),
                           (7093280, 0.5, 0.99, 1e-08), (7354384, 0.5, 0.99, 1e-08), (7357984, 0.5, 0.99, 1e-08),
                           (8005640, 0.5, 0.99, 1e-08), (8007688, 0.5, 0.99, 1e-08), (8011784, 0.5, 0.99, 1e-08),
                           (8271632, 0.5, 0.99, 1e-08), (8274208, 0.5, 0.99, 1e-08), (8567184, 0.5, 0.99, 1e-08),
                           (8568480, 0.5, 0.99, 1e-08), (8633488, 0.5, 0.99, 1e-08), (8637088, 0.5, 0.99, 1e-08),
                           (8641232, 0.5, 0.99, 1e-08), (8641888, 0.5, 0.99, 1e-08), (8659824, 0.5, 0.99, 1e-08),
                           (8660160, 0.5, 0.99, 1e-08), (8890120, 0.5, 0.99, 1e-08), (8892168, 0.5, 0.99, 1e-08),
                           (8953552, 0.5, 0.99, 1e-08), (8955360, 0.5, 0.99, 1e-08), (8957192, 0.5, 0.99, 1e-08),
                           (8961288, 0.5, 0.99, 1e-08), (9033712, 0.5, 0.99, 1e-08), (9034624, 0.5, 0.99, 1e-08),
                           (9053824, 0.5, 0.99, 1e-08), (9054288, 0.5, 0.99, 1e-08), (9111176, 0.5, 0.99, 1e-08),
                           (9112200, 0.5, 0.99, 1e-08), (9166408, 0.5, 0.99, 1e-08), (9166920, 0.5, 0.99, 1e-08),
                           (9180200, 0.5, 0.99, 1e-08), (9180456, 0.5, 0.99, 1e-08), (9194376, 0.5, 0.99, 1e-08),
                           (9196424, 0.5, 0.99, 1e-08), (9253576, 0.5, 0.99, 1e-08), (9254600, 0.5, 0.99, 1e-08),
                           (9268328, 0.5, 0.99, 1e-08), (9268840, 0.5, 0.99, 1e-08)],
    'twg_axpby': [   (100663296, '', 1.0, 0.0), (100663296, 'y', 1.0, 1.0), (1048576, '', 0.5, 0.0),
                     (1048576, '', 1.0, 0.0), (1048576, 'y', 0.5, 0.5), (1048576, 'y', 1.0, 1.0), (12288, '', 0.5, 0.0),
                     (12288, '', 1.0, 0.0), (12288, 'y', 0.5, 0.5), (12582912, '', 0.5, 0.0), (12582912, '', 1.0, 0.0),
                     (12582912, 'y', 0.5, 0.5), (12582912, 'y', 1.0, 1.0), (131072, '', 0.5, 0.0),
                     (131072, '', 1.0, 0.0), (131072, 'y', 0.5, 0.5), (131072, 'y', 1.0, 1.0), (1572864, 'y', 0.5, 0.5),
                     (16777216, '', 0.5, 0.0), (16777216, '', 1.0, 0.0), (16777216, 'y', 0.5, 0.5),
                     (16777216, 'y', 1.0, 1.0), (196608, '', 0.5, 0.0), (196608, '', 1.0, 0.0), (196608, 'y', 0.5, 0.5),
                     (196608, 'y', 1.0, 1.0), (2097152, '', 0.5, 0.0), (2097152, '', 1.0, 0.0),
                     (2097152, 'y', 0.5, 0.5), (2097152, 'y', 1.0, 1.0), (24576, 'y', 0.5, 0.5),
                     (25165824, '', 0.5, 0.0), (25165824, '', 1.0, 0.0), (25165824, 'y', 0.5, 0.5),
                     (25165824, 'y', 1.0, 1.0), (262144, '', 0.5, 0.0), (262144, '', 1.0, 0.0), (262144, 'y', 0.5, 0.5),
                     (262144, 'y', 1.0, 1.0), (3072, '', 1.0, 0.0), (3145728, '', 0.5, 0.0), (3145728, '', 1.0, 0.0),
                     (3145728, 'y', 0.5, 0.5), (3145728, 'y', 1.0, 1.0), (33554432, '', 1.0, 0.0),
                     (33554432, 'y', 1.0, 1.0), (393216, 'y', 0.5, 0.5), (4194304, '', 0.5, 0.0),
                     (4194304, '', 1.0, 0.0), (4194304, 'y', 0.5, 0.5), (4194304, 'y', 1.0, 1.0), (49152, '', 0.5, 0.0),
                     (49152, '', 1.0, 0.0), (49152, 'y', 0.5, 0.5), (50331648, '', 1.0, 0.0), (50331648, 'y', 1.0, 1.0),
                     (524288, '', 0.5, 0.0), (524288, '', 1.0, 0.0), (524288, 'y', 0.5, 0.5), (524288, 'y', 1.0, 1.0),
                     (592128, 'y', 1.0, 1.0), (6144, 'y', 0.5, 0.5), (6291456, '', 0.5, 0.0), (6291456, '', 1.0, 0.0),
                     (6291456, 'y', 0.5, 0.5), (6291456, 'y', 1.0, 1.0), (65536, '', 0.5, 0.0), (65536, '', 1.0, 0.0),
                     (65536, 'y', 0.5, 0.5), (65536, 'y', 1.0, 1.0), (67108864, '', 1.0, 0.0),
                     (67108864, 'y', 1.0, 1.0), (768, '', 1.0, 0.0), (786432, '', 0.5, 0.0), (786432, '', 1.0, 0.0),
                     (786432, 'y', 0.5, 0.5), (786432, 'y', 1.0, 1.0), (8388608, '', 0.5, 0.0), (8388608, '', 1.0, 0.0),
                     (8388608, 'y', 0.5, 0.5), (8388608, 'y', 1.0, 1.0), (98304, 'y', 0.5, 0.5)],
    'twg_bias_lrelu_fwd': [   (1024, 256, 0, 'bias'), (1024, 256, 1, 'bias+mask'), (1024, 256, 1, 'bias+planes+mask'),
                              (1048576, 16, 0, 'bias'), (1048576, 16, 1, 'bias+mask'),
                              (1048576, 16, 1, 'bias+planes+mask'), (12288, 256, 0, 'bias'),
                              (12288, 256, 1, 'bias+mask'), (12288, 256, 1, 'bias+planes+mask'),
                              (131072, 64, 0, 'bias'), (16, 1, 0, 'bias'), (16, 256, 1, 'bias'),
                              (16384, 128, 0, 'bias'), (16384, 128, 1, 'bias+mask'),
                              (16384, 128, 1, 'bias+planes+mask'), (196608, 64, 0, 'bias'),
                              (196608, 64, 1, 'bias+mask'), (196608, 64, 1, 'bias+planes+mask'), (2048, 256, 0, 'bias'),
                              (2097152, 16, 0, 'bias'), (256, 256, 0, 'bias'), (256, 256, 1, 'bias+mask'),
                              (262144, 32, 0, 'bias'), (262144, 32, 1, 'bias+mask'),
                              (262144, 32, 1, 'bias+planes+mask'), (3072, 256, 0, 'bias'), (3072, 256, 1, 'bias+mask'),
                              (3072, 256, 1, 'bias+planes+mask'), (3145728, 16, 0, 'bias'),
                              (3145728, 16, 1, 'bias+mask'), (3145728, 16, 1, 'bias+planes+mask'),
                              (32768, 128, 0, 'bias'), (4096, 256, 0, 'bias'), (4096, 256, 1, 'bias+mask'),
                              (4096, 256, 1, 'bias+planes+mask'), (48, 1, 0, 'bias'), (48, 256, 1, 'bias'),
                              (49152, 128, 0, 'bias'), (49152, 128, 1, 'bias+mask'),
                              (49152, 128, 1, 'bias+planes+mask'), (512, 256, 0, 'bias'), (524288, 32, 0, 'bias'),
                              (65536, 64, 0, 'bias'), (65536, 64, 1, 'bias+mask'), (65536, 64, 1, 'bias+planes+mask'),
                              (768, 256, 0, 'bias'), (768, 256, 1, 'bias+mask'), (786432, 32, 0, 'bias'),
                              (786432, 32, 1, 'bias+mask'), (786432, 32, 1, 'bias+planes+mask'),
                              (8192, 256, 0, 'bias')],
    'twg_copy_cols': [(9, 65792, 0, 98304, 0, 65792), (9, 98304, 0, 65792, 0, 65792)],
    'twg_dragan_xhat': [(16, 12288), (16, 192), (16, 196608), (16, 3072), (16, 48), (16, 49152), (16, 768)],
    'twg_fanout_bwd': [   (16, 12288, 'gds+gdt+ge2+gl_s+gl_t'), (16, 192, 'gds+gdt+ge2+gl_s+gl_t'),
                          (16, 196608, 'gds+gdt+ge2+gl_s+gl_t'), (16, 3072, 'gds+gdt+ge2+gl_s+gl_t'),
                          (16, 48, 'gds+gdt+ge2+gl_s+gl_t'), (16, 49152, 'gds+gdt+ge2+gl_s+gl_t'),
                          (16, 768, 'gds+gdt+ge2+gl_s+gl_t')],
    'twg_fanout_fwd': [(16, 12288), (16, 192), (16, 196608), (16, 3072), (16, 48), (16, 49152), (16, 768)],
    'twg_gan_losses': [(16,)],
    'twg_gan_losses_bwd': [(16, 'g0+g1'), (16, 'g1'), (16, 'g2+g3+g4+g5'), (16, 'g4+g5')],
    'twg_grad_penalty': [   (16, 12288, 0), (16, 192, 0), (16, 196608, 0), (16, 3072, 0), (16, 48, 0), (16, 49152, 0),
                            (16, 768, 0)],
    'twg_l1_groups': [(2, 65536)],
    'twg_lrelu_bwd': [(12288,), (2097152,), (4096,), (4194304,), (8388608,)],
    'twg_lrelu_bwd_colsum': [   (1024, 256, 0, 0, 0, 1, 'ref'), (1024, 256, 1, 0, 0, 1, 'ref+mask+out'),
                                (1048576, 16, 0, 0, 0, 1, 'ref'), (1048576, 16, 1, 0, 0, 1, 'ref+mask+out'),
                                (1048576, 16, 1, 0, 0, 1, 'ref+mask+out+planes'),
                                (1048576, 16, 1, 0, 0, 1, 'ref+mask+planes'), (1048576, 32, 0, 0, 0, 1, 'ref+planes'),
                                (1048576, 32, 1, 0, 0, 1, 'ref+mask+out'),
                                (1048576, 32, 1, 0, 0, 1, 'ref+mask+out+planes'),
                                (1048576, 32, 1, 0, 0, 1, 'ref+mask+planes'),
                                (1048576, 32, 1, 256, 256, 1, 'ref+mask+planes'), (12288, 256, 0, 0, 0, 1, 'ref'),
                                (12288, 256, 1, 0, 0, 1, 'ref+mask+out'), (131072, 128, 0, 0, 0, 1, 'ref+planes'),
                                (131072, 64, 0, 0, 0, 1, 'ref'), (16, 256, 1, 0, 0, 1, 'ref+out'),
                                (16384, 128, 0, 0, 0, 1, 'ref'), (16384, 128, 1, 0, 0, 1, 'ref+mask+out'),
                                (16384, 128, 1, 0, 0, 1, 'ref+out+planes'), (16384, 128, 1, 0, 0, 1, 'ref+planes'),
                                (16384, 256, 0, 0, 0, 1, 'ref+planes'), (16384, 256, 1, 0, 0, 1, 'ref+out+planes'),
                                (16384, 256, 1, 0, 0, 1, 'ref+planes'), (16384, 256, 1, 32, 32, 1, 'ref+planes'),
                                (196608, 128, 0, 0, 0, 0, 'ref+planes'), (196608, 128, 0, 0, 0, 1, 'ref+planes'),
                                (196608, 128, 1, 0, 0, 0, 'ref+planes'), (196608, 128, 1, 0, 0, 1, 'ref+planes'),
                                (196608, 128, 1, 64, 64, 0, 'ref+planes'), (196608, 128, 1, 64, 64, 1, 'ref+planes'),
                                (196608, 64, 0, 0, 0, 1, 'ref'), (196608, 64, 1, 0, 0, 0, 'ref+planes'),
                                (196608, 64, 1, 0, 0, 1, 'ref+mask+out'), (196608, 64, 1, 0, 0, 1, 'ref+planes'),
                                (2048, 256, 0, 0, 0, 1, 'ref'), (2097152, 16, 0, 0, 0, 1, 'ref'),
                                (2097152, 32, 0, 0, 0, 1, 'ref+planes'), (256, 256, 0, 0, 0, 1, 'ref'),
                                (256, 256, 1, 0, 0, 1, 'ref+mask+out'), (262144, 32, 0, 0, 0, 1, 'ref'),
                                (262144, 32, 1, 0, 0, 1, 'ref+mask+out'),
                                (262144, 32, 1, 0, 0, 1, 'ref+mask+out+planes'),
                                (262144, 32, 1, 0, 0, 1, 'ref+mask+planes'), (262144, 64, 0, 0, 0, 1, 'ref+planes'),
                                (262144, 64, 1, 0, 0, 1, 'ref+mask+out'),
                                (262144, 64, 1, 0, 0, 1, 'ref+mask+out+planes'),
                                (262144, 64, 1, 0, 0, 1, 'ref+mask+planes'),
                                (262144, 64, 1, 128, 128, 1, 'ref+mask+planes'), (3072, 256, 0, 0, 0, 1, 'ref'),
                                (3072, 256, 1, 0, 0, 1, 'ref+mask+out'), (3145728, 16, 0, 0, 0, 1, 'ref'),
                                (3145728, 16, 1, 0, 0, 0, 'ref+mask+planes'), (3145728, 16, 1, 0, 0, 1, 'ref+mask+out'),
                                (3145728, 16, 1, 0, 0, 1, 'ref+mask+planes'), (3145728, 32, 0, 0, 0, 0, 'ref+planes'),
                                (3145728, 32, 0, 0, 0, 1, 'ref+planes'), (3145728, 32, 1, 0, 0, 0, 'ref+mask+planes'),
                                (3145728, 32, 1, 0, 0, 1, 'ref+mask+planes'),
                                (3145728, 32, 1, 256, 256, 0, 'ref+mask+planes'),
                                (3145728, 32, 1, 256, 256, 1, 'ref+mask+planes'), (32768, 128, 0, 0, 0, 1, 'ref'),
                                (32768, 256, 0, 0, 0, 1, 'ref+planes'), (4096, 256, 0, 0, 0, 1, 'ref'),
                                (4096, 256, 1, 0, 0, 1, 'ref+mask+out'), (4194304, 16, 0, 0, 0, 1, 'ref+planes'),
                                (48, 1, 0, 0, 0, 1, 'ref'), (48, 256, 1, 0, 0, 1, 'ref+out'),
                                (49152, 128, 0, 0, 0, 1, 'ref'), (49152, 128, 1, 0, 0, 0, 'ref+planes'),
                                (49152, 128, 1, 0, 0, 1, 'ref+mask+out'), (49152, 128, 1, 0, 0, 1, 'ref+planes'),
                                (49152, 256, 0, 0, 0, 0, 'ref+planes'), (49152, 256, 0, 0, 0, 1, 'ref+planes'),
                                (49152, 256, 1, 0, 0, 0, 'ref+planes'), (49152, 256, 1, 0, 0, 1, 'ref+planes'),
                                (49152, 256, 1, 32, 32, 0, 'ref+planes'), (49152, 256, 1, 32, 32, 1, 'ref+planes'),
                                (512, 256, 0, 0, 0, 1, 'ref'), (524288, 32, 0, 0, 0, 1, 'ref'),
                                (524288, 64, 0, 0, 0, 1, 'ref+planes'), (65536, 128, 0, 0, 0, 1, 'ref+planes'),
                                (65536, 128, 1, 0, 0, 1, 'ref+out+planes'), (65536, 128, 1, 0, 0, 1, 'ref+planes'),
                                (65536, 128, 1, 64, 64, 1, 'ref+planes'), (65536, 64, 0, 0, 0, 1, 'ref'),
                                (65536, 64, 1, 0, 0, 1, 'ref+mask+out'), (65536, 64, 1, 0, 0, 1, 'ref+out+planes'),
                                (65536, 64, 1, 0, 0, 1, 'ref+planes'), (768, 256, 0, 0, 0, 1, 'ref'),
                                (768, 256, 1, 0, 0, 1, 'ref+mask+out'), (786432, 32, 0, 0, 0, 1, 'ref'),
                                (786432, 32, 1, 0, 0, 0, 'ref+mask+planes'), (786432, 32, 1, 0, 0, 1, 'ref+mask+out'),
                                (786432, 32, 1, 0, 0, 1, 'ref+mask+planes'), (786432, 64, 0, 0, 0, 0, 'ref+planes'),
                                (786432, 64, 0, 0, 0, 1, 'ref+planes'), (786432, 64, 1, 0, 0, 0, 'ref+mask+planes'),
                                (786432, 64, 1, 0, 0, 1, 'ref+mask+planes'),
                                (786432, 64, 1, 128, 128, 0, 'ref+mask+planes'),
                                (786432, 64, 1, 128, 128, 1, 'ref+mask+planes'), (8192, 256, 0, 0, 0, 1, 'ref')],
    'twg_mbstd_bwd': [(16, 16, 256, 384, 1), (48, 16, 256, 384, 3)],
    'twg_mbstd_bwd2': [(16, 16, 256, 384, 1)],
    'twg_mbstd_fwd': [(16, 16, 256, 384, 1, ''), (48, 16, 256, 384, 3, '')],
    'twg_pool2': [   (16, 128, 128, 3, 0.25, 'out'), (16, 128, 128, 64, 0.25, 'out'),
                     (16, 128, 128, 64, 0.25, 'out+planes'), (16, 16, 16, 256, 0.25, 'out'),
                     (16, 16, 16, 256, 0.25, 'out+planes'), (16, 16, 16, 3, 0.25, 'out'),
                     (16, 256, 256, 3, 0.25, 'out'), (16, 256, 256, 32, 0.25, 'out'),
                     (16, 256, 256, 32, 0.25, 'out+planes'), (16, 32, 32, 256, 0.25, 'out'),
                     (16, 32, 32, 256, 0.25, 'out+planes'), (16, 32, 32, 3, 0.25, 'out'),
                     (16, 64, 64, 128, 0.25, 'out'), (16, 64, 64, 128, 0.25, 'out+planes'),
                     (16, 64, 64, 3, 0.25, 'out'), (16, 8, 8, 256, 0.25, 'out'), (16, 8, 8, 3, 0.25, 'out'),
                     (32, 128, 128, 3, 0.25, 'out'), (32, 128, 128, 64, 0.25, 'out'),
                     (32, 128, 128, 64, 0.25, 'out+planes'), (32, 16, 16, 256, 0.25, 'out'),
                     (32, 16, 16, 256, 0.25, 'out+planes'), (32, 16, 16, 3, 0.25, 'out'),
                     (32, 256, 256, 3, 0.25, 'out'), (32, 256, 256, 32, 0.25, 'out'),
                     (32, 256, 256, 32, 0.25, 'out+planes'), (32, 32, 32, 256, 0.25, 'out'),
                     (32, 32, 32, 256, 0.25, 'out+planes'), (32, 32, 32, 3, 0.25, 'out'),
                     (32, 64, 64, 128, 0.25, 'out'), (32, 64, 64, 128, 0.25, 'out+planes'),
                     (32, 64, 64, 3, 0.25, 'out'), (32, 8, 8, 256, 0.25, 'out'), (32, 8, 8, 256, 0.25, 'out+planes'),
                     (32, 8, 8, 3, 0.25, 'out'), (48, 128, 128, 3, 0.25, 'out'), (48, 128, 128, 64, 0.25, 'out'),
                     (48, 128, 128, 64, 0.25, 'out+planes'), (48, 16, 16, 256, 0.25, 'out'),
                     (48, 16, 16, 256, 0.25, 'out+planes'), (48, 16, 16, 3, 0.25, 'out'),
                     (48, 256, 256, 3, 0.25, 'out'), (48, 256, 256, 32, 0.25, 'out'),
                     (48, 256, 256, 32, 0.25, 'out+planes'), (48, 32, 32, 256, 0.25, 'out'),
                     (48, 32, 32, 256, 0.25, 'out+planes'), (48, 32, 32, 3, 0.25, 'out'),
                     (48, 64, 64, 128, 0.25, 'out'), (48, 64, 64, 128, 0.25, 'out+planes'),
                     (48, 64, 64, 3, 0.25, 'out'), (48, 8, 8, 256, 0.25, 'out'), (48, 8, 8, 3, 0.25, 'out'),
                     (64, 128, 128, 3, 1.0, 'out'), (64, 128, 128, 64, 0.25, 'out+planes'),
                     (64, 16, 16, 256, 0.25, 'out+planes'), (64, 16, 16, 3, 1.0, 'out'), (64, 256, 256, 3, 1.0, 'out'),
                     (64, 256, 256, 32, 0.25, 'out+planes'), (64, 32, 32, 256, 0.25, 'out+planes'),
                     (64, 32, 32, 3, 1.0, 'out'), (64, 64, 64, 128, 0.25, 'out+planes'), (64, 64, 64, 3, 1.0, 'out'),
                     (64, 8, 8, 256, 0.25, 'out+planes'), (64, 8, 8, 3, 1.0, 'out')],
    'twg_scale_by_dev': [(1, 1.0)],
    'twg_scale_groups2': [(65536, -1.0, 'gl0+gl1'), (65536, 1.0, 'gl0+gl1')],
    'twg_scale_rows': [   (16, 12288, 'scalar'), (16, 192, 'scalar'), (16, 196608, 'scalar'), (16, 3072, 'scalar'),
                          (16, 48, 'scalar'), (16, 49152, 'scalar'), (16, 768, 'scalar')],
    'twg_sum_scalars': [(10, 1.0), (6, 1.0), (8, 1.0)],
    'twg_upsample2': [   (16, 128, 128, 3, 0.25), (16, 128, 128, 32, 0.25), (16, 16, 16, 256, 0.25),
                         (16, 16, 16, 3, 0.25), (16, 32, 32, 128, 0.25), (16, 32, 32, 3, 0.25), (16, 4, 4, 256, 0.25),
                         (16, 4, 4, 3, 0.25), (16, 64, 64, 3, 0.25), (16, 64, 64, 64, 0.25), (16, 8, 8, 256, 0.25),
                         (16, 8, 8, 3, 0.25), (32, 128, 128, 3, 0.25), (32, 128, 128, 3, 1.0), (32, 128, 128, 32, 0.25),
                         (32, 16, 16, 256, 0.25), (32, 16, 16, 3, 0.25), (32, 16, 16, 3, 1.0), (32, 32, 32, 128, 0.25),
                         (32, 32, 32, 3, 0.25), (32, 32, 32, 3, 1.0), (32, 4, 4, 256, 0.25), (32, 4, 4, 3, 0.25),
                         (32, 4, 4, 3, 1.0), (32, 64, 64, 3, 0.25), (32, 64, 64, 3, 1.0), (32, 64, 64, 64, 0.25),
                         (32, 8, 8, 256, 0.25), (32, 8, 8, 3, 0.25), (32, 8, 8, 3, 1.0), (48, 128, 128, 3, 0.25),
                         (48, 128, 128, 32, 0.25), (48, 16, 16, 256, 0.25), (48, 16, 16, 3, 0.25),
                         (48, 32, 32, 128, 0.25), (48, 32, 32, 3, 0.25), (48, 4, 4, 256, 0.25), (48, 4, 4, 3, 0.25),
                         (48, 64, 64, 3, 0.25), (48, 64, 64, 64, 0.25), (48, 8, 8, 256, 0.25), (48, 8, 8, 3, 0.25),
                         (64, 128, 128, 3, 1.0), (64, 16, 16, 3, 1.0), (64, 32, 32, 3, 1.0), (64, 4, 4, 3, 1.0),
                         (64, 64, 64, 3, 1.0), (64, 8, 8, 3, 1.0)],
    'twg_upsample_concat': [   (64, 128, 128, 32, 32, 32, 'out'), (64, 128, 128, 32, 32, 32, 'planes'),
                               (64, 128, 128, 32, 32, 64, 'planes'), (64, 16, 16, 256, 256, 32, 'out'),
                               (64, 16, 16, 256, 256, 32, 'planes'), (64, 16, 16, 256, 256, 64, 'planes'),
                               (64, 32, 32, 128, 128, 32, 'out'), (64, 32, 32, 128, 128, 32, 'planes'),
                               (64, 32, 32, 128, 128, 64, 'planes'), (64, 4, 4, 256, 256, 32, 'out'),
                               (64, 4, 4, 256, 256, 32, 'planes'), (64, 4, 4, 256, 256, 64, 'planes'),
                               (64, 64, 64, 64, 64, 32, 'out'), (64, 64, 64, 64, 64, 32, 'planes'),
                               (64, 64, 64, 64, 64, 64, 'planes'), (64, 8, 8, 256, 256, 32, 'out'),
                               (64, 8, 8, 256, 256, 32, 'planes'), (64, 8, 8, 256, 256, 64, 'planes')],
    'twg_upsample_concat_bwd': [   (64, 128, 128, 32, 32, 32), (64, 16, 16, 256, 256, 32), (64, 32, 32, 128, 128, 32),
                                   (64, 4, 4, 256, 256, 32), (64, 64, 64, 64, 64, 32), (64, 8, 8, 256, 256, 32)]}
PRODUCT_ELEMENTWISE_KEYS = {(entry,) + key for entry, keys in PRODUCT_ELEMENTWISE.items() for key in keys}


def cdiv(a, b):
  return -(-a // b)


def vec_geom(C):
  """(G, V) of vec_geom in twg_common.cuh, None for the two-pass widths."""
  if C % 4:
    return None
  q = C // 4
  if q <= 32:
    return (q, 1) if q & (q - 1) == 0 else None
  return (32, q // 32) if q % 32 == 0 and q // 32 in (1, 2, 4) else None


def colsum_plain_geom(rows, C):
  """(R, nb) of k_colsum for any C (twg_colsum always takes it)."""
  blocks = min(cdiv(rows, 256), 4 * 132)
  chunk = cdiv(rows, blocks)
  Cw = 1
  while Cw < C and Cw < 256:
    Cw <<= 1
  return cdiv(chunk, 256 // Cw), cdiv(rows, chunk)


def colsum_geom(rows, C, poolW=0, rows_route=False):
  """(R, nb) of a column sum: the terms one thread adds serially and the partial blocks add_partials adds in series, for
  k_colsum (odd C), k_lrelu_bwd_colsum_pool_rows (rows_route) and k_lrelu_bwd_colsum_vec, with their host-side grids."""
  gm = vec_geom(C)
  if gm is None:
    return colsum_plain_geom(rows, C)
  gpb = 256 // gm[0]
  if rows_route:
    img_rows = rows // poolW
    rpb = max(1, cdiv(img_rows, 8 * 132))
    return rpb * cdiv(poolW, gpb), cdiv(img_rows, rpb)
  blocks = max(1, min(cdiv(rows, gpb * 16), 8 * 132))
  chunk = cdiv(rows, blocks)
  return cdiv(chunk, gpb), cdiv(rows, chunk)


def pool_rows_route(C, lrelu_on, poolW, out, planes):
  gm = vec_geom(C)
  return bool(poolW and lrelu_on and planes and not out and gm and gm[1] == 1 and poolW >= 2 * (256 // gm[0]))


def penalty_geom(per):
  """(chunk, nb) of twg_grad_penalty's sums of squares: each sample's per_sample terms in nb blocks of chunk terms."""
  blocks = min(cdiv(per, 256 * 8), 64)
  chunk = cdiv(per, blocks)
  return chunk, cdiv(per, chunk)


def grid_for(n, per_thread=4):
  """Blocks of grid_for in twg_common.cuh: 256 threads, `per_thread` items each, at most 16 blocks per SM (132 SMs)."""
  return max(1, min(cdiv(n, 256 * per_thread), 132 * 16))


# cases beside the product's: routes the default flags never launch (twg_colsum, the two-pass odd widths of the fused
# column sum, the scalar pool / join kernels and the scalar backward of the join, Adam with a host step size, a leaky-ReLU
# backward whose length is not a multiple of 4), and the optional --loss_architecture terms at 16 pairs (3 logits each),
# both signs, with a hinge margin, scale_rows as the WGAN-GP penalty scales its gradient (no device scalar), and the
# losses of the unbatched passes (twg_sigmoid_ce on 16 logits per label, twg_l1 on a 256x256 cycle loss at 16 pairs; both
# also with accumulate and without a gradient)
EXTRA_ELEMENTWISE = {
    ('twg_colsum', 48, 1, 0), ('twg_colsum', 4096, 257, 0), ('twg_colsum', 786432, 32, 1), ('twg_colsum', 12288, 256, 1),
    ('twg_lrelu_bwd_colsum', 48, 1, 1, 0, 0, 1, 'ref+out'), ('twg_lrelu_bwd_colsum', 4096, 257, 1, 0, 0, 0, 'ref+out'),
    ('twg_lrelu_bwd_colsum', 4096, 257, 0, 0, 0, 1, ''),
    ('twg_pool2', 4, 16, 16, 3, 0.25, 'out'), ('twg_pool2', 4, 16, 16, 6, 1.0, 'out'),
    ('twg_upsample_concat', 4, 8, 8, 3, 6, 2, 'out'), ('twg_upsample_concat_bwd', 4, 8, 8, 3, 6, 2),
    ('twg_adam', 100003, 0.5, 0.99, 1e-08), ('twg_lrelu_bwd', 100003),
    ('twg_scale_rows', 16, 12288, ''),
    ('twg_sigmoid_ce', 16, 1.0, 0, 'grad'), ('twg_sigmoid_ce', 16, 0.0, 0, 'grad'), ('twg_sigmoid_ce', 1000, 1.0, 1, ''),
    ('twg_l1', 3145728, 0, 'grad'), ('twg_l1', 12288, 1, 'grad'), ('twg_l1', 1000, 0, ''),
}
for _kind in (0, 1, 2):
  for _sign, _margin in ((1.0, 0.0), (-1.0, 0.0), (1.0, 1.0), (-1.0, 1.0)):
    EXTRA_ELEMENTWISE |= {('twg_logit_mean', 48, _sign, _margin, _kind), ('twg_logit_mean_bwd', 48, _sign, _margin, _kind)}
