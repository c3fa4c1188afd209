"""The pipe-aware static timing model of tools/sass_time.py: the opcode -> pipe classifier on the opcodes of the two filter
walkers' round loops, and the scheduler on three hand-made sequences."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tools'))
import sass_time  # noqa: E402

# one line per opcode form that occurs in the round loops of k_mix_walk2 and k_mix_walk2c (CUDA 12.9, sm_90a)
WALKER_LOOP_SASS = {
    'alu': ['LOP3.LUT P4, RZ, R12, UR11, RZ, 0xc0, !PT', 'ISETP.EQ.OR P0, PT, R28, RZ, P4', 'SEL R30, R16, R11, !P4',
            '@!P4 LEA R12, R3, 0x1e00, 0x4', '@!P4 VIADD R33, R0, 0x200', '@!P4 IADD3 R19, R12, UR10, RZ',
            '@!P4 FSEL R10, R5, -1.00000001504746621988e+30, P0', 'PRMT R27, R12, 0x1045, R27',
            'FSETP.GT.AND P2, PT, R31, R28.reuse, PT', 'PLOP3.LUT P2, PT, P2, PT, PT, 0x8, 0x0', 'VOTE.ANY R19, PT, P0',
            'SHF.R.W.U32 R19, R19, UR13, R19', 'VIMNMX3.U32 R39, R30, UR14, R39, PT', 'VIMNMX.U32 R6, R6, 0x40, PT',
            'MOV R4, 0x2'],
    'fp32': ['FADD R36, R29, R34', 'FFMA R29, R29, 3.1999999919207766652e-05, R10', 'FMUL R2, R2, R3',
             'HFMA2.MMA R42, -RZ, RZ, 0, 5.9604644775390625e-08'],
    'imad': ['@!P4 IMAD R45, R15, UR6, R6.reuse', '@!P4 IMAD.WIDE.U32 R32, R33, 0x10, R22', 'IMAD.MOV.U32 R26, RZ, RZ, R28',
             'IMAD.SHL.U32 R15, R31, 0x8, RZ', 'IMAD.U32 R30, RZ, RZ, UR12', 'IMAD.IADD R3, R3, 0x1, R4'],
    'uni': ['UIADD3 UR12, -UR11, URZ, URZ', 'ULOP3.LUT UR11, UR11, UR12, URZ, 0xc0, !UPT', 'UPOPC UR14, UR11',
            'USHF.R.W.U32 UR15, UR12, UR13, UR12', 'ULEA UR12, UR15, 0x1, 0x1', 'UMOV UR12, UR4', 'VOTEU.ANY UR12, UPT, P2',
            'UISETP.NE.AND UP0, UPT, UR4, URZ, UPT', 'USEL UR4, UR5, UR6, UP0', 'UPLOP3.LUT UP0, UPT, UP0, UPT, UPT, 0x80, 0x0',
            'UFLO.U32 UR4, UR5'],
    'lsu': ['@!P0 STS.64 [R11], R26', 'LDS.64 R28, [R28]', 'LDS.U8 R27, [R8]', 'LDS.U16 R12, [R12]', 'LDS.128 R12, [R48]',
            '@P0 STG.E desc[UR16][R36.64], R8', '@!P4 LDGSTS.E.BYPASS.128 [R19], desc[UR16][R32.64]'],
    'ctl': ['NOP', 'LDGDEPBAR', 'DEPBAR.LE SB0, 0x8', '@!P4 BRA P1, 0x53e0', 'WARPSYNC.ALL'],
}


def test_every_walker_opcode_has_a_pipe():
    for pipe, lines in WALKER_LOOP_SASS.items():
        for text in lines:
            assert sass_time.pipe_of(text) == pipe, text


def test_unknown_opcode_is_an_error():
    with pytest.raises(KeyError):
        sass_time.pipe_of('FROBNICATE R0, R1')
    with pytest.raises(KeyError):
        sass_time.schedule([sass_time.ins('@P0 XYZZY.U32 R0, R1')])


def test_never_executed_filler_costs_one_slot():
    assert sass_time.issue_of('@!PT LDS RZ, [RZ]') == ('ctl', (1.0, 1.0))


def test_same_pipe_independent():
    # 8 independent ALU-pipe instructions: two cycles each for a lone warp, whatever their stall counts say
    T, total = sass_time.schedule([sass_time.ins('LOP3.LUT R%d, R%d, R20, R21, 0x96, !PT' % (k, k)) for k in range(8)])
    assert T == 16 and total == {'alu': 16}
    # without the issue table: the stall counts alone
    assert sass_time.schedule([sass_time.ins('LOP3.LUT R0, R0, R20, R21, 0x96, !PT')] * 8, pipes=False)[0] == 8
    # FP32: one per cycle
    assert sass_time.schedule([sass_time.ins('FADD R%d, R%d, R20' % (k, k)) for k in range(8)])[0] == 8
    # IMAD: its pipe takes one every two cycles
    assert sass_time.schedule([sass_time.ins('IMAD R%d, R%d, R20, R21' % (k, k)) for k in range(8)])[0] == 15


def test_two_pipes_interleaved():
    lop = sass_time.ins('LOP3.LUT R0, R0, R20, R21, 0x96, !PT')
    # ALU : FFMA and ALU : IMAD, 1:1 -- three cycles per pair (measured 2.9 and 3.0)
    assert sass_time.schedule([lop, sass_time.ins('FFMA R1, R1, R22, R23')] * 4)[0] == 12
    assert sass_time.schedule([lop, sass_time.ins('IMAD R1, R1, R22, R23')] * 4)[0] == 12
    # ALU : uniform -- the uniform datapath runs beside the vector pipes: 2.5 cycles per pair (measured 2.5)
    T, total = sass_time.schedule([lop, sass_time.ins('ULOP3.LUT UR4, UR4, UR5, URZ, 0xc0, !UPT')] * 4)
    assert T == pytest.approx(10.0)
    assert total['alu'] == 8 and total['uni'] == pytest.approx(9.6)


def test_scoreboard_bound():
    # LDS -> (scoreboard 0, 30 cycles) -> consumer: the pipes do not matter
    seq = [sass_time.ins('LDS.64 R28, [R28]', wbar=0), sass_time.ins('FADD R36, R29, R34', wait=1), sass_time.ins('FADD R1, R1, R2')]
    assert sass_time.schedule(seq)[0] == 32
    assert sass_time.schedule(seq, pipes=False)[0] == 32
    # a stall count above the issue cost stands
    assert sass_time.schedule([sass_time.ins('PRMT R27, R12, 0x1045, R27', stall=5), sass_time.ins('FADD R1, R1, R2')])[0] == 6
