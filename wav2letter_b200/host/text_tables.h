// text_tables.h — the device tables of one text pipeline (w2l_text_device_create): built on the host by
// host/text_pipeline.cpp from the pipeline's own Dictionary and splitWrd, uploaded and read by csrc/text_eval.cu.
#pragma once

#include <stdint.h>

#include <vector>

namespace w2l {

enum TextCriterion { kTextOther = 0, kTextCtc = 1, kTextAsg = 2, kTextSeq2Seq = 3 };

struct TextTablesHost {
  int criterion = kTextOther, replabel = 0;
  // token indices with a role in the path -> letters transform, -1 where the dictionary has none
  int blank = -1, eos = -1, pad = -1, sil = -1, surround = -1;
  int sep = -1;                          // letter id of the word separator, -1 if no letter equals it (or it is empty)
  std::vector<int8_t> role;              // [N] 0 ordinary, k > 0 the replabel <k>, -1 a token splitWrd refuses to spell
  std::vector<int32_t> ltrOff, ltr;      // CSR [N + 1] / [..]: token -> letter ids (tknIdx2Ltr's strings, one id per string)
  std::vector<int32_t> byteOff;          // CSR [letters + 1]: letter id -> its bytes, for exact word comparison
  std::vector<uint8_t> bytes;
};

// uploads the tables (one allocation); nullptr with the error text set on failure (csrc/text_eval.cu)
void* textDeviceUpload(const TextTablesHost& h, void* stream);
// the TextCriterion of an uploaded handle (csrc/text_eval.cu)
int textDeviceCriterion(const void* dev_text);

}  // namespace w2l
