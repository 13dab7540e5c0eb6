/*
 * feiscan_prog.h — binary layout of a compiled predicate program (the `prog` argument of
 * fei_scan_* in feiscan.h).  Built on the host by fei_b200/program.py from a SearchQuery
 * (memdir_tools/search.py:21-95) or MemoryFilter list (memdir_tools/filter.py:20-109).
 *
 * One program = up to 32 queries evaluated in one pass over the corpus.  A query is the AND
 * of its conditions (search.py:309-331; filter.py:80-107).  Every string-valued condition is
 * one output bit of a multi-output byte DFA attached to the field it reads
 * (fei_b200/regexc): all conditions on the same field share one automaton, so a field is
 * read once no matter how many queries look at it.  Patterns whose DFA is refused go to the field's position automaton
 * (fei_prog_nfa) instead, which owns the field's bits above its DFA's.
 *
 * Little-endian; offsets are bytes from the start of the blob; every section is 16-byte
 * aligned so tables can be staged into shared memory with 1-D bulk copies (cp.async.bulk).
 */
#ifndef FEISCAN_PROG_H_
#define FEISCAN_PROG_H_
#include <stdint.h>

#define FEI_PROG_MAGIC   0x50494546u   /* "FEIP" */
#define FEI_PROG_VERSION 1u
#define FEI_PROG_VERSION_NFA 2u        /* written only by programs that carry at least one position automaton (fei_prog_nfa):
                                          content (off_body_nfa), a header slot (fei_prog_slot.off_val_nfa), flags or a name
                                          field (off_head_nfa) */
#define FEI_PROG_VERSION_CTR 3u        /* written only by programs whose content position automaton has counters
                                          (fei_prog_nfa_ctr); every other program keeps version 1 or 2 */
#define FEI_MAX_QUERIES  32
#define FEI_MAX_SLOTS    16

/* condition kinds */
enum {
  FEI_C_CONST      = 0,  /* bit = constant truth value (host-evaluated, e.g. content without with_content) */
  FEI_C_BODY       = 1,  /* output `bit` of the body DFA           (content, search.py:103-104)           */
  FEI_C_SLOT       = 2,  /* output `bit` of header slot `ref`'s value DFA                                  */
  FEI_C_FLAGS      = 3,  /* output `bit` of the flags DFA          (search.py:105-106, filter.py:92-93)    */
  FEI_C_NAME       = 4,  /* output `bit` of name-field `ref` DFA: 0 filename, 1 unique_id, 2 hostname      */
  FEI_C_DATE_CMP   = 5,  /* wall-clock microseconds `cmp_op` i64   (search.py:107-108, :166-234)           */
  FEI_C_FOLDER_SET = 6,  /* (set64 >> folder_id) & 1               (host-evaluated per distinct folder); with
                            off_set_words != 0 the set is that bitmap instead (folder ids of 64 and above)       */
  FEI_C_STATUS_SET = 7,  /* (set64 >> status_id) & 1                                                        */
  FEI_C_RECBITS    = 8,  /* aux column `ref` of the corpus (fei_corpus_set_aux): one host-computed verdict byte per
                            record, for values only Python can judge (per-record dateutil parses of Due / Created /
                            Modified / DeletedDate headers, search.py:126-130)                                     */
  FEI_C_TS_CMP     = 9   /* filename timestamp (int) `cmp_op` i64  (metadata "timestamp", search.py:134-137)       */
};
/* FEI_C_NAME refs: 0 filename, 1 unique_id, 2 hostname (spans of the stored file name), and two strings the kernels
 * format from the meta columns: 3 = str(metadata["timestamp"]) (decimal digits), 4 = str(metadata["date"]) =
 * "YYYY-MM-DD HH:MM:SS" of datetime.fromtimestamp(ts) (filter.py:94-95; text operators of search.py:148-163 on `date`) */
#define FEI_NAME_FIELDS 5
enum { FEI_CMP_GT = 0, FEI_CMP_LT = 1, FEI_CMP_GE = 2, FEI_CMP_LE = 3, FEI_CMP_EQ = 4, FEI_CMP_NE = 5 };

typedef struct fei_prog_hdr {            /* 96 bytes */
  uint32_t magic, version, total_bytes;
  uint32_t n_queries;
  uint32_t n_conds, off_conds;           /* fei_prog_cond[n_conds]                                   */
  uint32_t off_queries;                  /* fei_prog_query[n_queries]                                */
  uint32_t n_slots, off_slots;           /* fei_prog_slot[n_slots]                                   */
  uint32_t off_key_dfa;                  /* fei_prog_dfa over header keys, one output bit per slot   */
  uint32_t off_body_dfa;                 /* 0 = no content condition                                 */
  uint32_t off_flags_dfa;
  uint32_t off_name_dfa[3];
  uint32_t head_mask;                    /* queries that have at least one non-body condition        */
  uint32_t body_mask;                    /* queries that have at least one body condition            */
  uint32_t slot_mask;                    /* queries that read at least one header slot                */
  uint32_t name_mask;                    /* queries that read filename / id / hostname                */
  uint32_t head_bytes;                   /* everything before the content automaton (which is serialised last): the part the
                                            head kernels copy into shared memory; 0 = unknown (do not stage)              */
  uint32_t off_meta_dfa[2];              /* name fields 3 and 4: automata over the formatted timestamp / date strings        */
  uint32_t off_body_nfa;                 /* version 2 or 3: fei_prog_nfa of the content patterns too large for the body DFA; 0 = none
                                            (version 3: present, with a fei_prog_nfa_ctr behind it) */
  uint32_t off_head_nfa;                 /* version 2 or 3: fei_prog_head_nfa (position automata of flags and the name fields); 0 = none */
} fei_prog_hdr;

/* Position automaton (bit-parallel NFA, fei_b200/regexc compile_positions), for content patterns whose DFA is too
 * large, and for the patterns of a head field (header slot, flags, name field) whose DFA is refused.  A value is stepped per code point over a W-word bit vector D of positions (bit 0: the virtual start, set before
 * the first character only):
 *     ctx = 1 << (prev_kind * 5 + kind(c))           kinds: 0 start / end, 1 '\n', 2 word, 3 Unicode-only word, 4 other
 *     acc |= OR over accept groups a, not end-only:  (D & src_a) != 0 && (ctx_a & ctx)  ->  bit_a
 *     D    = (((D << 1) & SHIFT) | (D & SELF) | OR over follow groups g: (D & src_g) != 0 && (ctx_g & ctx) -> dst_g) & B[class(c)]
 * and at the end with next kind 0, every accept group counted; the empty string is the reset vector finished at once.  Output
 * bits are first_bit .. first_bit + n_patterns - 1 of the field's verdict; the field's DFA, when it has one, owns the bits below
 * first_bit (the body DFA next to a content automaton is class-indexed and not sticky).  Every table is 16-byte aligned and the
 * tables are contiguous from off_ascii (table_bytes): one bulk copy stages them.  The sections of head fields (slots, flags,
 * names, fei_prog_head_nfa) lie inside [0, head_bytes), so the head kernels stage them with the rest of the head; the content
 * one lies behind it. */
typedef struct fei_prog_nfa {            /* 64 bytes */
  uint32_t n_words;                      /* W: 1, 2, 4 or 8 32-bit words per position vector                               */
  uint32_t n_pos;                        /* positions (bits) in use, the start bit included; <= 32 * W                      */
  uint32_t n_classes, n_ranges, n_follow, n_accept, n_patterns, first_bit;
  uint32_t off_ascii;                    /* uint16[128]: class | kind << 8 of each ASCII code point                         */
  uint32_t off_range_lo;                 /* uint32[n_ranges]: first code point of each non-ASCII range, ascending, [0] = 0x80 */
  uint32_t off_range_ck;                 /* uint16[n_ranges]: class | kind << 8 of each range                               */
  uint32_t off_cls_b;                    /* uint32[n_classes][W]: B, the positions whose leaf holds the class                */
  uint32_t off_masks;                    /* uint32[3][W]: SHIFT, SELF, START                                                 */
  uint32_t off_follow;                   /* uint32[n_follow][2W + 1]: src[W], dst[W], ctx mask                               */
  uint32_t off_accept;                   /* uint32[n_accept][W + 2]: src[W], ctx mask, output bit | end-only << 8             */
  uint32_t table_bytes;                  /* from off_ascii to the end of the accept table                                     */
} fei_prog_nfa;
#define FEI_NFA_MAX_CLASSES 128
#define FEI_NFA_MAX_RANGES  4096
#define FEI_NFA_MAX_GROUPS  64           /* follow groups, and accept groups, each */

/* Counters of the content position automaton (fei_b200/regexc compile_positions_counted): in a version-3 program, and only
 * there, this descriptor lies right behind the content fei_prog_nfa (at off_body_nfa + 64, before its tables); head fields
 * never have one.  Counter position P with bound k stands for a whole repeat `C{1,k}` of one character class: besides the
 * follow step, P stays set while C keeps matching and fewer than k code points have passed since its newest entry:
 *     entered = F[P];  D'[P] = B[class(c)][P] && (entered || (D[P] && age_P < k));  age_P = entered ? 1 : age_P + 1
 * with F = Follow(D, ctx) as above (every other bit is F & B[class(c)]); ages start at 0.  P is never in SELF and never
 * the start bit. */
typedef struct fei_prog_nfa_ctr {        /* 16 bytes */
  uint32_t n_counters;                   /* 1 .. FEI_NFA_MAX_COUNTERS                                                         */
  uint32_t off_counters;                 /* uint32[n_counters][2]: position, bound k >= 1; inside the section's tables        */
  uint32_t reserved[2];
} fei_prog_nfa_ctr;
#define FEI_NFA_MAX_COUNTERS 8

/* Position automata of flags and the name fields (fei_prog_hdr.off_head_nfa, inside [0, head_bytes)).  0 = the field has none;
 * a field with an automaton and no DFA has off_flags_dfa / off_name_dfa / off_meta_dfa 0. */
typedef struct fei_prog_head_nfa {       /* 32 bytes */
  uint32_t off_flags_nfa;
  uint32_t off_name_nfa[FEI_NAME_FIELDS];   /* indexed like FEI_C_NAME refs */
  uint32_t reserved[2];
} fei_prog_head_nfa;

typedef struct fei_prog_dfa {            /* 64 bytes; tables follow at the given offsets            */
  uint32_t n_states, n_cols;             /* n_cols == 256: byte-indexed rows; else class-indexed     */
                                         /* entry (s, col) lives at trans[s * row_stride + col]       */
  uint32_t start;
  uint32_t n_acc;                        /* states 0 .. n_acc-1 are exactly those with out != 0       */
  uint32_t off_trans, trans_bytes;       /* uint16[n_states * n_cols]                                 */
  uint32_t off_out, off_endout;          /* uint32[n_states] each                                     */
  uint32_t off_cls;                      /* uint8[256] byte -> column (class-indexed tables only)     */
  uint32_t n_outputs;
  uint32_t empty_acc;                    /* result mask for the empty string: out[start]|endout[start] */
  uint32_t table_bytes;                  /* trans + out + endout + cls, contiguous from off_trans     */
  uint32_t row_stride;                   /* entries per row; chosen so row_stride/2 is odd: consecutive
                                            states start in different shared-memory banks              */
  uint32_t sticky;                       /* 0: not sticky.  Else 1 + id of the absorbing "matched" state (0xFFFFFFFF: sticky
                                            but nothing can match): out[] is all zero, the verdict is endout[final state]     */
  uint32_t reserved[2];
} fei_prog_dfa;

typedef struct fei_prog_cond {           /* 32 bytes */
  uint8_t kind, ref, bit, negate;
  uint8_t if_missing;                    /* FEI_C_SLOT, header absent (and slot not empty_if_missing): 0 / 1 = the result;
                                            2 = the NEXT condition is the fallback field (filter.py:90-95: header, else
                                            flags / metadata); when the header is present the next condition is skipped */
  uint8_t cmp_op;
  uint8_t pad[2];
  int64_t i64;
  uint64_t set64;
  uint32_t off_set_words;                /* FEI_C_FOLDER_SET only: 0 = the set is set64 (folder ids 0..63).  Else the byte offset of
                                            the set as a bitmap, uint32_t[n_set_words], folder id k = bit k % 32 of word k / 32; ids
                                            at or above 32 * n_set_words are outside the set.  16-byte aligned and inside
                                            [0, head_bytes), so the head kernels stage it with the conditions.  program.py writes it
                                            only when the set holds a folder id of 64 or above; set64 then carries ids 0..63 too. */
  uint32_t n_set_words;                  /* ceil((largest folder id in the set + 1) / 32) */
} fei_prog_cond;

typedef struct fei_prog_query { uint32_t cond_begin, cond_end, reserved0, reserved1; } fei_prog_query;

typedef struct fei_prog_slot {           /* 16 bytes */
  uint32_t mode;                         /* 0: first key with key.lower()==field.lower(), last value of that exact key (search.py:121-132)
                                            1: exact key, last value (search.py:117-118 "Status"; filter.py:90-91)
                                            2: every key: OR over the values of the headers dict (utils.py:333-336, the legacy
                                               substring search); the key pattern of such a slot matches every key                      */
  uint32_t off_val_dfa;                  /* 0 = the slot has only a position automaton                                                   */
  uint32_t empty_if_missing;             /* 1: an absent header reads as "" (headers.get("Status", ""), search.py:118)                   */
  uint32_t off_val_nfa;                  /* version 2 or 3: fei_prog_nfa of the slot's patterns its DFA cannot hold; 0 = none; at least
                                            one of off_val_dfa / off_val_nfa is set                                                     */
} fei_prog_slot;

#endif /* FEISCAN_PROG_H_ */
