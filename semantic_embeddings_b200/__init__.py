"""H100-native hot path of cvjena/semantic-embeddings: training of hierarchy-based semantic image
embeddings (CNN -> L2-normalise -> 1-cosine loss against a fixed class-embedding matrix) and the
all-pairs retrieval distance matrix, as hand-written sm_90a CUDA behind a C ABI
(include/se_b200.h, libse_b200.so).  Host modules mirror the reference's Python interface:

  utils.py              build_network, l2norm, inv_correlation, nn_accuracy, get_lr_schedule  (reference utils.py)
  sgdr_callback.py      SGDR                                                                    (reference sgdr_callback.py)
  evaluate_retrieval.py pairwise_retrieval                                                      (reference evaluate_retrieval.py)
  models/               plainnet, cifar_resnet, wide_residual_network, resnet50                 (reference models/)
  engine.py             the layer-list executor that replaces Keras' compile/fit/predict
"""
__version__ = '0.1'
