// Opcodes of se_run_ops (include/se_b200.h).  Argument packing per op is documented in
// semantic_embeddings_b200/engine.py (the only producer) and api.cu (the only consumer).
#pragma once
enum {
  SE_OP_CONV_FWD = 1,
  SE_OP_CONV_DGRAD = 2,
  SE_OP_CONV_WGRAD = 3,
  SE_OP_BN_STATS = 4,
  SE_OP_BN_FWD_TRAIN = 5,
  SE_OP_BN_FWD_INFER = 6,
  SE_OP_BN_BWD = 7,
  SE_OP_SHORTCUT_BWD = 8,
  SE_OP_AVGPOOL_FWD = 9,
  SE_OP_AVGPOOL_BWD = 10,
  SE_OP_MAXPOOL_FWD = 11,
  SE_OP_MAXPOOL_BWD = 12,
  SE_OP_GAP_FWD = 13,
  SE_OP_GAP_BWD = 14,
  SE_OP_ADD_FWD = 15,
  SE_OP_ADD_BWD = 16,
  SE_OP_HEAD = 17,
  SE_OP_XENT = 18,
  SE_OP_MEMSET = 19,             /* p[0] = pointer, p[1] = bytes; i[0] bit 0: gradient memory -- join the side / comm streams first */
  SE_OP_SGD_PREPARE = 20,
  SE_OP_SGD_APPLY = 21,
  SE_OP_TRANSPOSE_FILTERS = 22,
  SE_OP_CONV_BN_FWD = 23,
  SE_OP_ALLREDUCE = 24,
  SE_OP_ADAGRAD_APPLY = 25,
  SE_OP_LABELEMBED = 26,
  SE_OP_CENTER_LOSS = 27,
};
