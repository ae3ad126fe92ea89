"""tools/ncu_source_stalls.py -- per-source-line warp-stall breakdown of one kernel from an ncu capture.

   cuobjdump -xelf all cppnumericalsolvers_b200/libcno.so && nvdisasm -gi cno_api.sm_90a.cubin > gi.txt
   ncu -i prof.ncu-rep --page source --csv > source.csv          (capture made with --set full --import-source on)
   python tools/ncu_source_stalls.py gi.txt source.csv <mangled kernel name>

Joins the SASS addresses of ncu's source page with nvdisasm's inline line info (innermost file:line per instruction) and
prints, per source line, its share of all stall samples, the instructions executed (1e7) and the share of every stall
reason in percent of ALL samples.  Used for DESIGN.md 2.4."""
import re, csv, collections, sys
gi, src, fn = sys.argv[1:4]
txt=open(gi).read().split('\n')
start=[i for i,l in enumerate(txt) if l.startswith('.text.'+fn)][0]
chain=[]; amap={}; pending=[]
for l in txt[start+1:]:
    if l.startswith('//-----') : break
    m=re.match(r'\s*//## File "([^"]*)", line (\d+)', l)
    if m:
        pending.append((m.group(1).split('/')[-1], int(m.group(2)))); continue
    m=re.match(r'\s*/\*([0-9a-f]{4,})\*/\s+(.*);', l)
    if m:
        if pending: chain=pending; pending=[]
        amap[int(m.group(1),16)]=(chain, m.group(2))
rows=list(csv.reader(open(src)))
hdr=rows[1]; body=rows[2:]
ix={h:i for i,h in enumerate(hdr)}
base=int(body[0][ix['Address']],16)
keys=['stall_no_inst','stall_branch_resolving','stall_wait','stall_short_sb','stall_barrier','stall_not_selected','stall_selected','stall_long_sb']
agg=collections.defaultdict(lambda: collections.Counter())
for r in body:
    try: a=int(r[ix['Address']],16)-base
    except: continue
    ch=amap.get(a,([],''))[0]
    # innermost location
    loc=ch[0] if ch else ('?',0)
    for k in keys:
        try: agg[loc][k]+=int(r[ix[k]])
        except: pass
    agg[loc]['n']+=int(r[ix['# Samples']] or 0); agg[loc]['e']+=int(r[ix['Instructions Executed']] or 0)
tot=sum(v['n'] for v in agg.values())
print('total',tot)
print('%-28s %6s %6s | '%('loc','samp%','instr') + ' '.join(k[6:12].rjust(7) for k in keys))
for loc,v in sorted(agg.items(), key=lambda kv:-kv[1]['n'])[:45]:
    print('%-28s %6.2f %6.2f | '%(f'{loc[0]}:{loc[1]}',100*v['n']/tot, v['e']/1e7)+' '.join(('%7.2f'%(100*v[k]/tot)) for k in keys))
