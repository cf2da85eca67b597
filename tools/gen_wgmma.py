"""Writes the wgmma_m64nNk16 specialisations (N = 16, 32, ..., 256) between the GENERATED markers of
long-video-gan_b200/csrc/wgmma.cuh. One inline-asm statement per N: the accumulator list of an instruction is N / 2
registers long, and PTX wants it spelled out.   python tools/gen_wgmma.py"""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, 'long-video-gan_b200', 'csrc', 'wgmma.cuh')
BEGIN, END = '// ---- BEGIN GENERATED (tools/gen_wgmma.py)', '// ---- END GENERATED'


def block():
    lines = []
    for n in range(16, 257, 16):
        r = n // 2
        regs = '{' + ', '.join(f'%{i}' for i in range(r)) + '}'
        ins = [str(r + i) for i in range(7)]
        outs = ', '.join(f'LVG_D8({i})' for i in range(0, r, 8))
        kw = 'if' if n == 16 else 'else if'
        lines.append(f'    {kw} constexpr (N == {n}) LVG_WGMMA("{n}", "{regs}", "{ins[0]}", "{ins[1]}", "{ins[2]}", "{ins[3]}", "{ins[4]}", '
                     f'"{ins[5]}", "{ins[6]}", {outs});')
    return '\n'.join(lines)


def main():
    src = open(PATH).read()
    pat = re.compile(re.escape(BEGIN) + r'\n.*?' + re.escape(END), re.S)
    assert pat.search(src), 'markers not found'
    out = pat.sub(lambda _: BEGIN + '\n' + block() + '\n    ' + END, src)
    open(PATH, 'w').write(out)


if __name__ == '__main__':
    main()
