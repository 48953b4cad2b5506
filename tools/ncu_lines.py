"""Per-source-line summary of an ncu report (needs -lineinfo builds and --import-source on):
    python tools/ncu_lines.py prof.ncu-rep [top_n]
Prints the source lines with the most warp-stall samples / executed instructions and their average active threads."""
import csv
import subprocess
import sys

rep = sys.argv[1]
top = int(sys.argv[2]) if len(sys.argv) > 2 else 40
extra = []
for a in sys.argv[3:]:
    if a.startswith('--launch='):                      # which captured launch of the report (0-based)
        extra = ['--launch-skip', a.split('=')[1], '--launch-count', '1']
sys.argv = [a for a in sys.argv if not a.startswith('--launch=')]
out = subprocess.run(['ncu', '-i', rep] + extra + ['--page', 'source', '--print-source', 'cuda,sass', '--csv'],
                     capture_output=True, text=True).stdout
rows = list(csv.reader(out.splitlines()))
hdr = None
lines = []
cur = ''
want = sys.argv[3] if len(sys.argv) > 3 else '.cu'
for r in rows:
    if r and r[0] == 'File Path':
        cur = r[1]
        continue
    if r and r[0] == 'Line No':
        hdr = r
        continue
    if hdr and r and r[0].isdigit() and want in cur and len(r) == len(hdr):
        try:
            float(r[hdr.index('Instructions Executed')])
        except ValueError:
            continue
        lines.append(r)
ci = hdr.index('Instructions Executed')
ti = hdr.index('Thread Instructions Executed')
si = hdr.index('# Samples')
stall = [i for i, h in enumerate(hdr) if h.startswith('stall_') and 'Not Issued' not in h]
tot_i = sum(float(r[ci]) for r in lines)
tot_s = sum(float(r[si]) for r in lines)
print(f'total warp-instructions {tot_i:.3e}, samples {tot_s:.0f}')
lines.sort(key=lambda r: -float(r[si]))
for r in lines[:top]:
    inst, thr, smp = float(r[ci]), float(r[ti]), float(r[si])
    st = sorted(((float(r[i]), hdr[i][6:]) for i in stall), reverse=True)[:2]
    print(f'{int(r[0]):4d} samp {smp / tot_s * 100:5.1f}% inst {inst / tot_i * 100:5.1f}% thr {thr / max(inst, 1):4.1f} '
          f'{st[0][1]}:{st[0][0]:.0f} {st[1][1]}:{st[1][0]:.0f} | {r[1].strip()[:90]}')
