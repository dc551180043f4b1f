#!/bin/bash
# dis.sh <binary> -> /tmp/<name>.view (annotated SASS of range_lean_kernel)
b=$(realpath $1); n=$(basename $b)
d=$(mktemp -d); (cd $d && cuobjdump -xelf all $b >/dev/null 2>&1; nvdisasm -g -c *.cubin > /tmp/$n.sass)
python "$(dirname "$0")/sass_view.py" /tmp/$n.sass range_lean_kernel > /tmp/$n.view
rm -rf $d; wc -l /tmp/$n.view
