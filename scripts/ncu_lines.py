"""Join an ncu SASS-page CSV with nvdisasm line info of the built library: per-file / per-line / per-opcode shares.
usage: python scripts/ncu_lines.py gpurun_out/prof.ncu-rep 'rollout_kernel_warpILi72ELi2' [steps]"""
import collections, csv, os, re, subprocess, sys, tempfile
rep, kern = sys.argv[1], sys.argv[2]
steps = float(sys.argv[3]) if len(sys.argv) > 3 else 7577600.0
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
tmp = tempfile.mkdtemp()
subprocess.run(['cuobjdump', '-xelf', 'all', os.path.join(ROOT, 'serl_b200', 'libserl_b200.so')], cwd=tmp, capture_output=True)
sass = subprocess.run(['nvdisasm', '-c', '-g', os.path.join(tmp, 'rollout.sm_90a.cubin')], capture_output=True, text=True).stdout.split('\n')
start = [i for i, l in enumerate(sass) if l.startswith('.text.') and kern in l][0]
end = next((i for i in range(start + 1, len(sass)) if sass[i].startswith('//--------------------- .text.')), len(sass))
cur, ins = None, []
for l in sass[start:end]:
    m = re.match(r'\s*//## File "(.*)", line (\d+)', l)
    if m:
        cur = (m.group(1).split('/')[-1], int(m.group(2))); continue
    m = re.match(r'\s*/\*([0-9a-f]{4,})\*/\s+(.*?);', l)
    if m:
        ins.append((int(m.group(1), 16), m.group(2), cur))
csvtxt = subprocess.run(['ncu', '-i', rep, '--page', 'source', '--csv', '--print-source', 'sass'], capture_output=True, text=True).stdout
rows = list(csv.reader(csvtxt.splitlines()))
hdr, data = rows[1], rows[2:]
ia, iex, ismp, isrc = hdr.index('Address'), hdr.index('Instructions Executed'), hdr.index('# Samples'), hdr.index('Source')
base = int(data[0][ia], 16)
prof = {int(r[ia], 16) - base: (int(r[iex]), int(r[ismp])) for r in data}
F, FS, Ln, LS, O, OS = (collections.Counter() for _ in range(6))
for off, txt, c in ins:
    if off not in prof:
        continue
    ex, sm = prof[off]
    f = c[0] if c else '?'
    F[f] += ex; FS[f] += sm; Ln[c] += ex; LS[c] += sm
    t = txt.split()
    op = (t[1] if t[0].startswith('@') else t[0]).split('.')[0]
    O[op] += ex; OS[op] += sm
tot, ts = sum(F.values()), sum(FS.values())
print('instructions %d, warp-instr executed %.3e = %.0f thread-instr per env-step' % (len(ins), tot, tot * 32 / steps))
for f, v in F.most_common():
    print('%-28s exec %5.1f%% samples %5.1f%%' % (f, 100 * v / tot, 100 * FS[f] / ts))
print('--- opcodes')
for k, v in O.most_common(24):
    print('%-8s exec %5.1f%% per-step %6.0f samples %5.1f%%' % (k, 100 * v / tot, v * 32 / steps, 100 * OS[k] / ts))
print('--- top lines by samples')
for k, v in LS.most_common(16):
    print(k, 'samples %.2f%% exec %.2f%%' % (100 * v / ts, 100 * Ln[k] / tot))
for name in hdr:
    if name.startswith('stall_') and 'Not Issued' not in name:
        i = hdr.index(name); s = sum(int(r[i]) for r in data if r[i].isdigit())
        if s > 0.02 * ts:
            print(name, '%.1f%%' % (100 * s / ts))
