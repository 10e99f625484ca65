#!/bin/bash
# A/B sweeps on the C2 workload; prints views/s and per-stage ms/view.  Usage: bash profiles/sweep.sh [tiles|switches|streams]
# (scratch output goes to $SWEEP_DIR, default a fresh temporary directory)
# Switches (all default to the faster setting; each keeps the other implementation selectable for cross-checks):
#   LGS_SORT=lgs|cub            own radix sort | cub::DeviceRadixSort          LGS_TILE_RANGE=search|scan   lower_bound per tile | streaming
#   LGS_STAGING=cpasync|bulk    3 x cp.async | cp.async.bulk + mbarrier         LGS_BWD_REDUCE=smem|butterfly  backward warp reduction
#   LGS_VIEWS_AUTOGRAD=0|1      render_views direct | through the autograd Function     LGS_WPB=4|2|1  tiles per CTA
SWEEP_DIR=${SWEEP_DIR:-$(mktemp -d)}
run() {  # label, env..., -- bench args
  local label="$1"; shift
  env "$@" timeout 300 python bench.py --steps 20 --warmup 3 --no-e2e --no-cpu-baseline $EXTRA > "$SWEEP_DIR/sw.json" 2>"$SWEEP_DIR/sw.err" || { echo "FAIL $label"; tail -3 "$SWEEP_DIR/sw.err"; return; }
  python - "$label" "$SWEEP_DIR/sw.json" <<'PY'
import json,sys
d=json.load(open(sys.argv[2])); s=d['stages']
print(f"{sys.argv[1]:34s} views/s {d['value']:7.1f} ms/view {d['path_roofline']['ms_per_view']:.3f} D {d['workload_stats']['D']}  " +
      " ".join(f"{k[4:].replace('rasterize_','r').replace('_packed','').replace('sort_pairs_','sort')}={v['ms_per_view']:.3f}" for k,v in s.items()))
PY
}
what=${1:-switches}
if [ "$what" = tiles ]; then
  for t in 8x16 12x16 16x16 8x8; do EXTRA="--tile $t" run "tile $t" LGS_WPB=4; done
elif [ "$what" = streams ]; then
  for n in 1 2 3 4 6; do EXTRA="--streams $n" run "streams $n" LGS_WPB=4; done
else
  EXTRA="" run "defaults" LGS_WPB=4
  EXTRA="" run "LGS_SORT=cub" LGS_SORT=cub
  EXTRA="" run "LGS_TILE_RANGE=scan" LGS_TILE_RANGE=scan
  EXTRA="" run "LGS_STAGING=bulk" LGS_STAGING=bulk
  EXTRA="" run "LGS_BWD_REDUCE=butterfly" LGS_BWD_REDUCE=butterfly
  EXTRA="" run "LGS_VIEWS_AUTOGRAD=1" LGS_VIEWS_AUTOGRAD=1
  EXTRA="" run "LGS_WPB=2" LGS_WPB=2
fi
