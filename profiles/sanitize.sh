#!/bin/bash
# compute-sanitizer over a small slice of the GPU parity suite (SURVEY.md section 5: race detection / sanitizers).
# memcheck: out-of-bounds / misaligned accesses in every kernel the selected tests launch; racecheck: shared-memory hazards in
# the streaming kernels (mbarrier-synchronised bulk-copy rings, the TMA + wgmma kernels, the per-column radix select); synccheck:
# barrier / mbarrier misuse. Usage (on an H100): bash profiles/sanitize.sh [memcheck|racecheck|synccheck|all]
set -u
TOOL=${1:-all}
WIDE="(test_full_run_matches_reference and 2d_full]) or (test_sparse_estep_matches_float64_oracle and 0]) or (test_voxel_data_device_matches_host and 2-float32) or test_gene_cost_kl_matches_oracle or (test_kwargs_surface and large_K)"
NARROW="(test_single_estep_matches_float64_oracle and 2d_full and 0-) or (test_sparse_estep_matches_float64_oracle and 0]) or test_gene_cost_kl_matches_oracle"
# M-step kernels: the Jacobi solve (shared memory, block barriers), the low-rank apply, the ordered moment reduction
MSTEP="(spectrum_and_warm_starts and cutoff_straddle) or lowrank or rigid_moments or (one_mstep and (K65 or K33))"
JACOBI="spectrum_and_warm_starts and (clustered-15 or cutoff_straddle-64) or svi_blend_and_guidance"
# sparse top-k select: candidate-cap overflow, ties at tau, subnormals (racecheck / synccheck); 514 row blocks (memcheck)
SELECT="test_written_cap_ties_subnormals_against_replay and 1024-True"
MASKOFF="test_mask_off_above_512_row_blocks and 32"
# trajectory integration: control points tiled through shared memory (block barriers) and the event / step-rejection paths
PATH_TILED="test_inducing_points_above_the_shared_memory_tile"
PATH_MEM="test_inducing_points_above_the_shared_memory_tile or test_event_stops or (test_sparsevfc_field and 2)"
run() {  # tool, pytest args...
  local tool=$1; shift
  echo "=== compute-sanitizer --tool $tool : $*"
  compute-sanitizer --tool "$tool" --error-exitcode 9 --launch-timeout 0 python -m pytest -q -x "$@" 2>&1 | grep -E "passed|failed|ERROR SUMMARY|Race reported|hazard|Error:|error" | tail -12
  echo "exit code: ${PIPESTATUS[0]}"
}
if [ "$TOOL" = memcheck ] || [ "$TOOL" = all ]; then
  run memcheck tests/test_gpu_parity.py -k "$WIDE"
  run memcheck tests/test_gpu_gram.py -k "64-7000 or 257-4100 or 15-5000 or 3-900"
  run memcheck tests/test_gpu_shard.py -k "1]"
  run memcheck tests/test_gpu_shard_options.py -k "mapping_from_identical_state or svi_estep_from_identical_state"
  run memcheck tests/test_gpu_mstep.py -k "$MSTEP"
  run memcheck tests/test_gpu_posterior_select.py -k "$MASKOFF"
  run memcheck tests/test_gpu_morphopath.py -k "$PATH_MEM"
fi
if [ "$TOOL" = racecheck ] || [ "$TOOL" = all ]; then
  run racecheck tests/test_gpu_parity.py -k "$NARROW"
  run racecheck tests/test_gpu_gram.py -k "64-7000"
  run racecheck tests/test_gpu_mstep.py -k "$JACOBI"
  run racecheck tests/test_gpu_posterior_select.py -k "$SELECT"
  run racecheck tests/test_gpu_morphopath.py -k "$PATH_TILED"
fi
if [ "$TOOL" = synccheck ] || [ "$TOOL" = all ]; then
  run synccheck tests/test_gpu_parity.py -k "$NARROW"
  run synccheck tests/test_gpu_gram.py -k "64-7000"
  run synccheck tests/test_gpu_mstep.py -k "$JACOBI"
  run synccheck tests/test_gpu_posterior_select.py -k "$SELECT"
  run synccheck tests/test_gpu_morphopath.py -k "$PATH_TILED"
fi
