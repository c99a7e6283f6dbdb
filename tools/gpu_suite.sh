#!/bin/bash
# Runs the GPU test groups in separate processes (a trapped kernel kills its CUDA context, not the whole suite).
# usage: tools/gpu_suite.sh [group ...]   logs -> profile_out/suite_<group>.log
mkdir -p profile_out
groups=("$@")
[ ${#groups[@]} -eq 0 ] && groups=(conv_fwd fwd_b fwd_c fwd_d fwd_e conv_misc conv_dgrad conv_wgrad elementwise simota nms engine modeling iou fused optim streams fixed_order train_bn mosaic cnx_ops cnx_engine attention detr detr_dropout sparseinst strict yolox_convnext detr_criterion convnext_plan sparseinst_kernels sparseinst_criterion detr_kernels sparseinst_bwd sparseinst_encoder sparseinst_model detr_model headline_fwd headline_eval headline_dgrad headline_wgrad headline_probe headline_step)
for g in "${groups[@]}"; do
  case $g in
    conv_fwd)    sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and not 1x320 and not 16x64 and not 8x80x80'" ;;
    fwd_a)       sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and 1x32x32'" ;;
    fwd_b)       sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and 16x64x64x16'" ;;
    fwd_c)       sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and 16x64x64x64'" ;;
    fwd_d)       sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and 8x80x80'" ;;
    fwd_e)       sel="tests/test_conv_gpu.py -k 'test_conv_fwd_stats and 1x320'" ;;
    conv_misc)   sel="tests/test_conv_gpu.py -k 'slices or bias'" ;;
    conv_dgrad)  sel="tests/test_conv_gpu.py -k test_conv_dgrad" ;;
    conv_wgrad)  sel="tests/test_conv_gpu.py -k test_conv_wgrad" ;;
    elementwise) sel="tests/test_elementwise_gpu.py" ;;
    simota)      sel="tests/test_simota_gpu.py" ;;
    engine)      sel="tests/test_engine_gpu.py" ;;
    nms)         sel="tests/test_nms_gpu.py" ;;
    modeling)    sel="tests/test_modeling_gpu.py" ;;
    iou)         sel="tests/test_iou_loss_gpu.py" ;;
    streams)     sel="tests/test_streams_gpu.py" ;;
    fixed_order) sel="tests/test_fixed_order_gpu.py" ;;
    train_bn)    sel="tests/test_train_bn_gpu.py" ;;
    mosaic)      sel="tests/test_mosaic_gpu.py" ;;
    fused)       sel="tests/test_conv_gpu.py -k fused" ;;
    optim)       sel="tests/test_optim_gpu.py" ;;
    attention)   sel="tests/test_attention_gpu.py tests/test_attention_bwd_gpu.py" ;;
    detr)        sel="tests/test_detr_gpu.py" ;;
    detr_dropout) sel="tests/test_detr_dropout_gpu.py" ;;
    detr_criterion) sel="tests/test_detr_criterion_gpu.py" ;;
    strict)      sel="tests/test_strict_gpu.py" ;;
    yolox_convnext) sel="tests/test_yolox_convnext_gpu.py" ;;
    convnext_plan) sel="tests/test_convnext_plan_gpu.py" ;;
    sparseinst)  sel="tests/test_sparseinst_gpu.py" ;;
    sparseinst_kernels) sel="tests/test_sparseinst_kernels_gpu.py" ;;
    sparseinst_criterion) sel="tests/test_sparseinst_criterion_gpu.py" ;;
    sparseinst_bwd) sel="tests/test_sparseinst_bwd_gpu.py" ;;
    sparseinst_encoder) sel="tests/test_sparseinst_encoder_gpu.py" ;;
    sparseinst_model) sel="tests/test_sparseinst_model_gpu.py" ;;
    detr_model)  sel="tests/test_detr_model_gpu.py" ;;
    detr_kernels) sel="tests/test_detr_kernels_gpu.py" ;;
    headline_fwd)   sel="tests/test_headline_plan_gpu.py -k 'test_recording or test_fwd'" ;;
    headline_eval)  sel="tests/test_headline_plan_gpu.py -k test_eval_fwd" ;;
    headline_dgrad) sel="tests/test_headline_plan_gpu.py -k test_dgrad" ;;
    headline_wgrad) sel="tests/test_headline_plan_gpu.py -k test_wgrad" ;;
    headline_probe) sel="tests/test_headline_plan_gpu.py -k 'test_probe or test_spp'" ;;
    headline_step)  sel="tests/test_headline_plan_gpu.py -k 'test_batchnorm or test_head_bias or test_simota or test_focus or test_eval_batchnorm'" ;;
    cnx_ops)     sel="tests/test_convnext_gpu.py -k 'not engine and not block_against'" ;;
    cnx_engine)  sel="tests/test_convnext_gpu.py -k 'engine or block_against'" ;;
    *)           sel="$g" ;;
  esac
  echo "=== $g"
  eval timeout ${SUITE_TIMEOUT:-300} python -u -m pytest $sel -m gpu -q -x --durations=5 --timeout=120 --timeout-method=thread -p no:cacheprovider ${SUITE_ARGS:-} 2>&1 | tail -80 | cut -c1-400 > profile_out/suite_$g.log
  tail -4 profile_out/suite_$g.log
done
