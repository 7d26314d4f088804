#!/bin/bash
# SASS evidence per hot kernel (cuobjdump needs no GPU), written under the git-ignored tune/ directory:
#   tune/sass_<round>/<kernel>.txt = resource usage + the instructions that carry the design
#   (UBLKCP / SYNCS = bulk-copy engine + mbarrier, LDG.E.128 = 16-byte table records, multimem / STG.E.128 row stores).
set -e
R=${1:-r02}
SO=pytorch_volumetric_b200/csrc/libpvb.so
OUT=tune/sass_$R
mkdir -p "$OUT"
dump() {   # name, mangled-name regex, grep pattern
  local f="$OUT/$1.txt"
  { echo "# $1 -- cuobjdump -sass / -res-usage of $SO ($(date -u +%F))"
    cuobjdump -res-usage "$SO" 2>/dev/null | grep -A1 -E "$2" | grep -E "Function|REG" | head -4
    echo "# instruction count: $(cuobjdump -sass "$SO" 2>/dev/null | awk -v pat="$2" '$0 ~ "Function : " {f = ($0 ~ pat)} f' | grep -cE '^\s+/\*[0-9a-f]{4,}\*/')"
    echo "# opcode histogram (top 12)"
    cuobjdump -sass "$SO" 2>/dev/null | awk -v pat="$2" '$0 ~ "Function : " {f = ($0 ~ pat)} f' | grep -E '^\s+/\*[0-9a-f]{4,}\*/' \
      | sed -E 's/^\s+\/\*[0-9a-f]+\*\/\s+//; s/^@!?U?P[0-9T]+ //' | awk '{print $1}' | sed -E 's/\..*//' | sort | uniq -c | sort -rn | head -12
    echo "# selected instructions ($3)"
    cuobjdump -sass "$SO" 2>/dev/null | awk -v pat="$2" '$0 ~ "Function : " {f = ($0 ~ pat)} f' | grep -E "$3" | sed -E 's/\s+\/\* 0x[0-9a-f]+ \*\/$//' | head -24
  } > "$f"
  echo "$f: $(wc -l < "$f") lines"
}
dump grid_lookup_tma      'grid_lookup_tma_kernel'                'UBLKCP|SYNCS|LDG\.E\.128'
dump robot_serial         'robot_serial_kernelILi0'               'LDG\.E\.128|STG\.E.*128|MUFU\.RSQ|SHFL|LDS\.128'
dump robot_serial_mc      'robot_serial_kernelILi2'               'STG\.E.*STRONG\.SYS'
dump mesh_query           'mesh_query_kernel'                     'LDG\.E\.128|STG\.E\.128'
dump fk_serial            'fk_serial_kernel'                      'MUFU|STG\.E\.128'
dump compact_write        'compact_write_kernelIf'                'SHFL|STG'
