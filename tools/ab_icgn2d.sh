# A/B harness for icgn2d.cu: build variants in opencorr_b200/lib/variants/*.so (selected with OCB_LIB_PATH) and the
# OCB_ICGN2D_WPP knob
run() { python bench.py --no-cpu-baseline --steps 20 --config ${2:-B} 2>/dev/null | tail -1 | python -c "import sys,json; d=json.loads(sys.stdin.read()); print('$1', '${2:-B}', 'step_ms', round(d['ms_per_step'],4), 'icgn_ms', round(d['roofline']['kernel_ms'],4))"; }
for c in ${CONFIGS:-B}; do
run default $c
for v in opencorr_b200/lib/variants/*.so; do [ -f $v ] && OCB_LIB_PATH=$PWD/$v run $(basename $v .so) $c; done
done
